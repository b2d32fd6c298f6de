"""OLMo 2 on the CPU: ``debug-olmo2`` against ``transformers.Olmo2ForCausalLM`` with the same weights (logits, loss and
every gradient), the op's CPU path against the reference functions it composes, the registry's parameter counts
against the meta-device model, the HF config round trip and its refusals, an HF checkpoint loaded through
``--pretrained``, the layer's flat layout, DDP / FSDP over gloo against one process, the single-engine flags, gradient
accumulation, and the refusal of the tensor-parallel engines."""
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

OLMO2 = {   # id: (hidden, intermediate, layers, heads, kv heads, parameters)
    "allenai/OLMo-2-0425-1B": (2048, 8192, 16, 16, 16, 1_484_916_736),
    "allenai/OLMo-2-1124-7B": (4096, 11008, 32, 32, 32, 7_298_617_344),
    "allenai/OLMo-2-1124-13B": (5120, 13824, 40, 40, 40, 13_716_198_400),
    "allenai/OLMo-2-0325-32B": (5120, 27648, 64, 40, 8, 32_234_279_936),
}


# ---------------------------------------------------------------------------------------------------------------
# the ops' CPU paths
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("per_token", [False, True])
def test_olmo_qk_norm_rope_cpu_path_composes_reference(per_token):
    g = torch.Generator().manual_seed(0)
    B, S, nh, nkv, d = 2, 12, 4, 2, 16
    qkv = torch.randn(B, S, nh + 2 * nkv, d, generator=g) * 3
    q_w, k_w = torch.randn(nh * d, generator=g), torch.randn(nkv * d, generator=g)
    pos = torch.randint(0, 50, (B, S), generator=g) if per_token else torch.arange(S)
    cos, sin = ref.rope_tables(pos, d, 5e5)
    out = ops.olmo_qk_norm_rope_(qkv, q_w, k_w, cos, sin, nh, nkv, 1e-6)
    q = ref.rms_norm_one_rounding(qkv[:, :, :nh].reshape(B, S, nh * d), q_w, 1e-6).view(B, S, nh, d)
    k = ref.rms_norm_one_rounding(qkv[:, :, nh:nh + nkv].reshape(B, S, nkv * d), k_w, 1e-6).view(B, S, nkv, d)
    torch.testing.assert_close(out[:, :, :nh], ref.rope_apply(q, cos, sin))
    torch.testing.assert_close(out[:, :, nh:nh + nkv], ref.rope_apply(k, cos, sin))
    assert torch.equal(out[:, :, nh + nkv:], qkv[:, :, nh + nkv:])
    # full width: scaling one q head changes the other q heads' outputs (a per-head norm would not), and scaling
    # every q head together changes nothing
    scaled = qkv.clone()
    scaled[:, :, 0] *= 7.0
    out1 = ops.olmo_qk_norm_rope_(scaled, q_w, k_w, cos, sin, nh, nkv, 1e-6)
    assert (out1[:, :, 1:nh] - out[:, :, 1:nh]).abs().max() > 1e-2
    torch.testing.assert_close(out1[:, :, nh:nh + nkv], out[:, :, nh:nh + nkv])
    scaled = qkv.clone()
    scaled[:, :, :nh] *= 7.0
    out2 = ops.olmo_qk_norm_rope_(scaled, q_w, k_w, cos, sin, nh, nkv, 1e-6)
    torch.testing.assert_close(out2[:, :, :nh], out[:, :, :nh], rtol=1e-5, atol=1e-5)


def test_one_rounding_norm_and_norm_then_add_reference():
    g = torch.Generator().manual_seed(1)
    x = (torch.randn(64, 256, generator=g) * 4).bfloat16()
    r = torch.randn(64, 256, generator=g).bfloat16()
    w = (torch.randn(256, generator=g) * 2).bfloat16()
    xf = x.double()
    y64 = w.double() * xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + 1e-6)
    y = ref.rms_norm_one_rounding(x, w, 1e-6)
    assert y.dtype == torch.bfloat16
    # one rounding: within half a bf16 ulp of the exact value (plus the fp32 statistic's error)
    assert ((y.double() - y64).abs() <= y64.abs() * (2.0 ** -8 + 1e-6) + 1e-30).all()
    h = ref.rms_norm_add(x, r, w, 1e-6)
    assert torch.equal(h, (r.float() + y.float()).bfloat16())
    # the CPU op is the reference
    assert torch.equal(ops.rms_norm_add(x, r, w, 1e-6), h)


# ---------------------------------------------------------------------------------------------------------------
# the model against transformers
# ---------------------------------------------------------------------------------------------------------------
def _hf_olmo2(cfg, transformers):
    d = {k: v for k, v in to_hf_config_dict(cfg).items() if k not in ("model_type", "architectures", "torch_dtype")}
    hf_cfg = transformers.Olmo2Config(**d)
    hf_cfg._attn_implementation = "eager"
    return transformers.Olmo2ForCausalLM(hf_cfg).float().eval()


def _spread_debug_olmo2(cfg):
    """fp32 model whose norm gains are spread around a scale other than 1, so that every gain is visible in the
    output and the q/k gains sharpen attention away from uniform."""
    torch.manual_seed(0)
    mine = build_model(cfg, dtype=torch.float32, device="cpu")
    g = torch.Generator().manual_seed(3)
    with torch.no_grad():
        for layer in mine.model.layers:
            for n in (layer.self_attn.q_norm, layer.self_attn.k_norm):
                n.weight.copy_(3.0 * (1 + 0.3 * torch.randn(n.weight.shape, generator=g)))
            for n in (layer.post_attention_layernorm, layer.post_feedforward_layernorm):
                n.weight.copy_(0.5 * (1 + 0.3 * torch.randn(n.weight.shape, generator=g)))
    return mine


@pytest.mark.parametrize("tied", [False, True])
def test_debug_olmo2_matches_transformers_fp32(tied):
    transformers = pytest.importorskip("transformers")
    cfg = get_config("debug-olmo2", tie_word_embeddings=tied)
    assert cfg.arch == "olmo2" and cfg.full_qk_norm and cfg.post_norm and not cfg.qk_norm and cfg.head_dim == 128
    assert cfg.num_attention_heads != cfg.num_key_value_heads
    mine = _spread_debug_olmo2(cfg)
    hf = _hf_olmo2(cfg, transformers)
    missing, unexpected = hf.load_state_dict(mine.state_dict(), strict=False)
    assert not unexpected, unexpected
    assert all("rotary" in m or "inv_freq" in m for m in missing), missing   # names are HF's
    assert [n for n, _ in mine.named_parameters()] == [n for n, _ in hf.named_parameters()]   # and so is the order
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
    for key in ("q_norm", "k_norm", "post_attention_layernorm", "post_feedforward_layernorm"):
        assert any(key in n for n in names), key
    assert not any("input_layernorm" in n for n in names)
    layer = mine.model.layers[0]
    assert layer.self_attn.q_norm.weight.shape == (cfg.num_attention_heads * 128,)
    assert layer.self_attn.k_norm.weight.shape == (cfg.num_key_value_heads * 128,)
    for n, p in mine.named_parameters():
        want = hf_params[n].grad
        err = ((p.grad - want).norm() / want.norm()).item()
        assert err < 1e-4, (n, err)


# ---------------------------------------------------------------------------------------------------------------
# configs
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(OLMO2))
def test_registry_olmo2(name):
    h, i, l, nh, nkv, n = OLMO2[name]
    cfg = get_config(name)
    assert cfg.arch == "olmo2" and cfg.full_qk_norm and not cfg.qk_norm and cfg.head_dim == 128
    assert (cfg.vocab_size, cfg.hidden_size, cfg.intermediate_size, cfg.num_hidden_layers) == (100352, h, i, l)
    assert (cfg.num_attention_heads, cfg.num_key_value_heads, cfg.tie_word_embeddings) == (nh, nkv, False)
    assert (cfg.rope_theta, cfg.rms_norm_eps, cfg.max_position_embeddings) == (5e5, 1e-6, 4096)
    assert cfg.num_parameters() == n
    assert build_model(cfg, dtype=torch.bfloat16, device="meta").num_parameters() == n


def test_num_parameters_meta_and_transformers():
    cfg = get_config("debug-olmo2")
    assert build_model(cfg, dtype=torch.float32, device="meta").num_parameters() == cfg.num_parameters()
    transformers = pytest.importorskip("transformers")
    for name in list(OLMO2) + ["debug-olmo2"]:
        c = get_config(name)
        d = {k: v for k, v in to_hf_config_dict(c).items() if k not in ("model_type", "architectures", "torch_dtype")}
        with torch.device("meta"):
            hf = transformers.Olmo2ForCausalLM(transformers.Olmo2Config(**d))
        assert sum(p.numel() for p in hf.parameters()) == c.num_parameters(), name


def _write_config(tmp_path, d):
    (tmp_path / "config.json").write_text(json.dumps(d))
    return str(tmp_path)


@pytest.mark.parametrize("name", ["allenai/OLMo-2-1124-7B", "allenai/OLMo-2-0325-32B", "debug-olmo2"])
def test_hf_config_round_trip(tmp_path, name):
    cfg = get_config(name)
    d = to_hf_config_dict(cfg)
    assert d["model_type"] == "olmo2" and d["architectures"] == ["Olmo2ForCausalLM"]
    back = get_config(_write_config(tmp_path, d))
    assert back.to_dict() == {**cfg.to_dict(), "name": str(tmp_path)}
    transformers = pytest.importorskip("transformers")
    hf = transformers.Olmo2Config(**{k: v for k, v in d.items() if k not in ("model_type", "architectures")})
    assert hf.num_key_value_heads == cfg.num_key_value_heads and hf.tie_word_embeddings is False
    assert hf.rope_parameters["rope_theta"] == cfg.rope_theta and hf.rms_norm_eps == cfg.rms_norm_eps


def test_hf_config_layouts_and_refusals(tmp_path):
    d = to_hf_config_dict(get_config("debug-olmo2"))
    # transformers>=5 writes rope_parameters instead of rope_theta
    v5 = {k: v for k, v in d.items() if k != "rope_theta"}
    v5["rope_parameters"] = {"rope_theta": 5e5, "rope_type": "default"}
    cfg = get_config(_write_config(tmp_path, v5))
    assert cfg.rope_theta == 5e5 and cfg.rope_scaling is None and cfg.arch == "olmo2"
    for bad, key in (({"attention_bias": True}, "attention_bias"),
                     ({"rope_parameters": {"rope_theta": 5e5, "rope_type": "yarn", "factor": 8.0}}, "rope_parameters"),
                     ({"rope_scaling": {"rope_type": "linear", "factor": 2.0}}, "rope_scaling"),
                     ({"head_dim": 64}, "head_dim")):
        with pytest.raises(ValueError, match=key):
            get_config(_write_config(tmp_path, {**d, **bad}))
    # an explicit head_dim equal to hidden / heads is accepted
    assert get_config(_write_config(tmp_path, {**d, "head_dim": 128})).head_dim == 128
    with pytest.raises(ValueError, match="olmo3"):
        get_config(_write_config(tmp_path, {**d, "model_type": "olmo3"}))


def test_pretrained_hf_olmo2_checkpoint_loads(tmp_path):
    transformers = pytest.importorskip("transformers")
    pytest.importorskip("safetensors")
    from distributed_training_guide_b200.tools.load_hf import maybe_load_pretrained

    cfg = get_config("debug-olmo2")
    torch.manual_seed(5)
    hf = _hf_olmo2(cfg, transformers)
    with torch.no_grad():   # gains other than 1, so that loading them is visible
        for n, p in hf.named_parameters():
            if "norm" in n:
                p.uniform_(0.5, 2.0)
    hf.save_pretrained(str(tmp_path / "m"), safe_serialization=True)
    loaded_cfg = get_config(str(tmp_path / "m"))
    assert loaded_cfg.arch == "olmo2" and loaded_cfg.head_dim == 128 and loaded_cfg.full_qk_norm
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
def test_flat_order_holds_every_parameter_with_the_matrices_first():
    from distributed_training_guide_b200.parallel.flat import build_groups

    model = build_model(get_config("debug-olmo2"), dtype=torch.bfloat16, device="cpu")
    layer = model.model.layers[0]
    order = layer.flat_order
    assert set(order) == {n for n, _ in layer.named_parameters()} and len(order) == len(set(order))
    assert not any("input_layernorm" in n for n in order)
    named = dict(layer.named_parameters())
    dims = [named[n].dim() for n in order]
    assert dims == sorted(dims, reverse=True), "matrices first"
    assert order == ("self_attn.q_proj.weight", "self_attn.k_proj.weight", "self_attn.v_proj.weight",
                     "self_attn.o_proj.weight", "mlp.gate_proj.weight", "mlp.up_proj.weight", "mlp.down_proj.weight",
                     "post_attention_layernorm.weight", "post_feedforward_layernorm.weight",
                     "self_attn.q_norm.weight", "self_attn.k_norm.weight")
    assert layer.fused == {"qkv": order[:3], "gate_up": order[4:6]}
    assert all(named[n].numel() % 8 == 0 for n in order)
    groups = build_groups(model, "cpu", torch.bfloat16)
    assert len({id(p) for g in groups for p in g.params}) == len(list(model.parameters()))
    g = groups[1]
    assert [n.split(".", 3)[-1] for n in g.names] == list(order)
    # the fused q|k|v and gate|up views exist and span the adjacent matrices
    assert layer._fused["qkv"].data.shape == (512 + 2 * 256, 512)
    assert layer._fused["gate_up"].data.shape == (2 * 1024, 512)
    # a Llama layer's order is unchanged
    llama = build_model(get_config("debug-llama-gqa"), dtype=torch.bfloat16, device="meta")
    assert llama.model.layers[0].flat_order == (
        "self_attn.q_proj.weight", "self_attn.k_proj.weight", "self_attn.v_proj.weight", "self_attn.o_proj.weight",
        "mlp.gate_proj.weight", "mlp.up_proj.weight", "mlp.down_proj.weight", "input_layernorm.weight",
        "post_attention_layernorm.weight")


def test_layers_complete_the_stream_and_model_norm_finishes():
    """Every layer sees residual None and returns (h2, None); the forward equals composing the reference ops."""
    cfg = get_config("debug-olmo2")
    model = _spread_debug_olmo2(cfg)
    ids = torch.randint(0, cfg.vocab_size, (1, 32), generator=torch.Generator().manual_seed(4))
    m = model.model
    cos, sin = m.rotary_emb.tables(32, ids.device)
    x = m.embed_tokens(ids)
    for layer in m.layers:
        out, res = layer(x, None, cos, sin)
        assert res is None and out.shape == x.shape
        att = layer.self_attn
        qkv = ref.linear(x, torch.cat([att.q_proj.weight, att.k_proj.weight, att.v_proj.weight])).view(1, 32, 8, 128)
        qkv = ops.olmo_qk_norm_rope_(qkv, att.q_norm.weight, att.k_norm.weight, cos, sin, 4, 2, 1e-6)
        a = ref.attention(qkv[:, :, :4], qkv[:, :, 4:6], qkv[:, :, 6:]).reshape(1, 32, 512)
        h1 = ref.rms_norm_add(ref.linear(a, att.o_proj.weight), x, layer.post_attention_layernorm.weight, 1e-6)
        mlp = layer.mlp
        gu = ref.linear(h1, torch.cat([mlp.gate_proj.weight, mlp.up_proj.weight]))
        h2 = ref.rms_norm_add(ref.linear(ref.swiglu(gu), mlp.down_proj.weight), h1,
                              layer.post_feedforward_layernorm.weight, 1e-6)
        torch.testing.assert_close(out, h2)
        x = out
    with pytest.raises(AssertionError):
        m.layers[0](x, x, cos, sin)


# ---------------------------------------------------------------------------------------------------------------
# engines over gloo against one process
# ---------------------------------------------------------------------------------------------------------------
S_DIST, LR_DIST, B_GLOBAL = 256, 5e-3, 4


def _batch(vocab, step, rank, B=1):
    g = torch.Generator().manual_seed(1000 * step + rank)
    ids = torch.randint(0, vocab, (B, S_DIST), generator=g)
    return {"input_ids": ids, "labels": ids.clone()}


def _gains(model):
    out = []
    for l in model.model.layers:
        out.append(torch.cat([l.self_attn.q_norm.weight.detach().float(), l.self_attn.k_norm.weight.detach().float(),
                              l.post_attention_layernorm.weight.detach().float(),
                              l.post_feedforward_layernorm.weight.detach().float()]))
    return out


def _train_dist(rank, world, parallelism, steps):
    from distributed_training_guide_b200.engine import TrainEngine

    torch.manual_seed(0)
    per = B_GLOBAL // world
    eng = TrainEngine.create("debug-olmo2", parallelism=parallelism, batch_size=per, seq_length=S_DIST, device="cpu",
                             lr=LR_DIST)
    dp_rank = eng.strategy.dp_rank
    losses, gains = [], []
    for i in range(steps):
        parts = [_batch(eng.config.vocab_size, i, dp_rank * per + j) for j in range(per)]
        losses.append(float(eng.step({k: torch.cat([p[k] for p in parts]) for k in parts[0]})))
        if parallelism != "fsdp":   # FSDP holds shards; its gains are checked through the loss
            gains.append(_gains(eng.model))
    return losses, gains, eng.strategy.dp_size


def _single(steps):
    from distributed_training_guide_b200.engine import TrainEngine

    torch.manual_seed(0)
    eng = TrainEngine.create("debug-olmo2", parallelism="single", batch_size=B_GLOBAL, seq_length=S_DIST,
                             device="cpu", lr=LR_DIST)
    losses, gains = [], []
    for i in range(steps):
        parts = [_batch(eng.config.vocab_size, i, r) for r in range(B_GLOBAL)]
        losses.append(float(eng.step({k: torch.cat([p[k] for p in parts]) for k in parts[0]})))
        gains.append(_gains(eng.model))
    return losses, gains


@pytest.mark.parametrize("parallelism", ["ddp", "fsdp"])
def test_distributed_olmo2_matches_single_process(parallelism):
    steps, world = 3, 2
    res = run_distributed(_train_dist, world=world, args=(parallelism, steps), timeout=600)
    assert res[0][2] == world
    ref_losses, ref_gains = _single(steps)
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


@pytest.mark.parametrize("flags", [dict(fp8=True), dict(max_grad_norm=1.0), dict(checkpoint_activations=True),
                                   dict(document_masking=True)])
def test_single_engine_flags_train_olmo2(flags):
    """The flags a Llama run takes also train debug-olmo2: finite losses, and the gains get their updates."""
    from distributed_training_guide_b200.engine import TrainEngine

    torch.manual_seed(0)
    eng = TrainEngine.create("debug-olmo2", parallelism="single", batch_size=1, seq_length=128, device="cpu",
                             lr=LR_DIST, **flags)
    g0 = _gains(eng.model)
    for i in range(2):
        b = _batch(eng.config.vocab_size, i, 0)
        b = {k: v[:, :128] for k, v in b.items()}
        if flags.get("document_masking"):
            b["position_ids"] = torch.cat([torch.arange(50), torch.arange(78)])[None]
        assert math.isfinite(float(eng.step(b)))
    assert all(not torch.equal(a, b) for a, b in zip(g0, _gains(eng.model)))


def test_activation_checkpointing_gives_the_same_gradients():
    from distributed_training_guide_b200.parallel.flat import build_groups

    cfg = get_config("debug-olmo2")
    ids = torch.randint(0, cfg.vocab_size, (2, 64), generator=torch.Generator().manual_seed(6))
    grads = []
    for ckpt in (False, True):
        model = _spread_debug_olmo2(cfg)
        groups = build_groups(model, "cpu", torch.float32)
        for g in groups:
            g.zero_grad()
        model.activation_checkpointing = ckpt
        model(input_ids=ids, labels=ids).loss.backward()
        grads.append(torch.cat([g.grad.clone() for g in groups]))
    assert grads[0].abs().sum() > 0
    torch.testing.assert_close(grads[1], grads[0], rtol=1e-5, atol=1e-7)


def test_gradient_accumulation_matches_the_unaccumulated_step():
    """Two half batches with the loss halved accumulate into the flat gradient what one full batch writes."""
    from distributed_training_guide_b200.parallel.flat import build_groups

    cfg = get_config("debug-olmo2")
    model = _spread_debug_olmo2(cfg)
    groups = build_groups(model, "cpu", torch.float32)
    ids = torch.randint(0, cfg.vocab_size, (4, 64), generator=torch.Generator().manual_seed(7))
    for g in groups:
        g.zero_grad()
    model(input_ids=ids, labels=ids).loss.backward()
    full = torch.cat([g.grad.clone() for g in groups])
    for g in groups:
        g.zero_grad()
    for half in (ids[:2], ids[2:]):
        (model(input_ids=half, labels=half).loss / 2).backward()
    acc = torch.cat([g.grad.clone() for g in groups])
    assert full.abs().sum() > 0
    # fp32 sums in another order: compare as a whole, and element by element at a looser bound
    assert ((acc - full).norm() / full.norm()).item() < 1e-5
    torch.testing.assert_close(acc, full, rtol=1e-2, atol=1e-5)


@pytest.mark.parametrize("parallelism", ["tp", "2d"])
def test_tensor_parallel_engines_refuse_olmo2(parallelism):
    from distributed_training_guide_b200.engine import TrainEngine

    with pytest.raises(ValueError, match="full-width q/k norm"):
        TrainEngine.create("debug-olmo2", parallelism=parallelism, batch_size=1, seq_length=128, device="cpu",
                           tensor_parallel=1)


def _tp2(rank, world):
    from distributed_training_guide_b200.engine import TrainEngine

    try:
        TrainEngine.create("debug-olmo2", parallelism="2d", batch_size=1, seq_length=256, device="cpu",
                           tensor_parallel=2)
    except ValueError as e:
        return str(e)
    return None


def test_two_rank_tensor_parallel_refuses_olmo2():
    res = run_distributed(_tp2, world=2, args=(), timeout=300)
    assert all(r is not None and "full-width q/k norm" in r for r in res), res
