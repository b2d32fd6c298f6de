"""GPT-NeoX / Pythia on the CPU: ``debug-gpt-neox`` (head_dim 128, rotary 32) and ``debug-gpt-neox-d64`` (head_dim
64, rotary 16) against ``transformers.GPTNeoXForCausalLM`` with the same weights mapped through
``models.gpt_neox_layout`` (logits, loss and every gradient, tied and untied), the new ops' CPU paths, the registry's
parameter counts against the published Pythia totals and the meta-device models, the HF config round trip in both
key layouts and its refusals, an HF checkpoint loaded through ``--pretrained`` and written back by the consolidation
tool, the layer's flat layout and parallel residual, DDP / FSDP over gloo against one process, the single-engine
flags, gradient accumulation, and the refusal of the tensor-parallel engines."""
import dataclasses
import json
import math
import subprocess
import sys
from pathlib import Path
from types import SimpleNamespace

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from dist_utils import run_distributed
from distributed_training_guide_b200 import ops
from distributed_training_guide_b200.models import build_model, get_config, gpt_neox_layout, to_hf_config_dict
from distributed_training_guide_b200.ops import reference as ref

PYTHIA = {   # size: (hidden, intermediate, layers, heads, vocab, published parameter count)
    "70m": (512, 2048, 6, 8, 50304, 70_426_624),
    "160m": (768, 3072, 12, 12, 50304, 162_322_944),
    "410m": (1024, 4096, 24, 16, 50304, 405_334_016),
    "1.4b": (2048, 8192, 24, 16, 50304, 1_414_647_808),
    "6.9b": (4096, 16384, 32, 32, 50432, 6_857_302_016),
    "12b": (5120, 20480, 36, 40, 50688, 11_846_072_320),
}
DEBUG = ["debug-gpt-neox", "debug-gpt-neox-d64"]


# ---------------------------------------------------------------------------------------------------------------
# the ops' CPU paths
# ---------------------------------------------------------------------------------------------------------------
def test_layer_norm2_gelu_partial_rope_and_parallel_out_cpu_paths():
    g = torch.Generator().manual_seed(0)
    x = (torch.randn(16, 64, generator=g) * 3 + 1).bfloat16()
    r = torch.randn(16, 64, generator=g).bfloat16()
    w1, b1, w2, b2 = (torch.randn(64, generator=g).bfloat16() for _ in range(4))
    y1, y2, h = ops.layer_norm2(x, r, w1, b1, w2, b2, 1e-5)
    assert torch.equal(h, x + r)
    assert torch.equal(y1, ref.layer_norm(x + r, w1, b1, 1e-5)) and torch.equal(y2, ref.layer_norm(x + r, w2, b2, 1e-5))
    y1, y2, h = ops.layer_norm2(x, None, w1, b1, w2, b2, 1e-5)
    assert h is x and torch.equal(y1, ref.layer_norm(x, w1, b1, 1e-5))
    t = torch.linspace(-8, 8, 4096)
    torch.testing.assert_close(ops.gelu(t), F.gelu(t), rtol=0, atol=0)
    assert torch.equal(ops.gelu(t.bfloat16()), F.gelu(t.bfloat16().float()).bfloat16())
    # partial rotary: the first 32 of 128 elements of the q and k heads rotate, the rest and v are untouched
    qkv = torch.randn(2, 8, 6, 128, generator=g)
    cos, sin = ref.rope_tables(torch.arange(8), 32, 1e4)
    out = ops.rope_qkv_(qkv.clone(), cos, sin, 4, 32)
    assert torch.equal(out[..., 32:], qkv[..., 32:]) and torch.equal(out[:, :, 4:], qkv[:, :, 4:])
    assert torch.equal(out[:, :, :4, :32], ref.rope_apply(qkv[:, :, :4, :32], cos, sin))
    assert not torch.equal(out[:, :, :4, :32], qkv[:, :, :4, :32])
    full_cos, full_sin = ref.rope_tables(torch.arange(8), 128, 1e4)
    assert torch.equal(ops.rope_qkv_(qkv.clone(), full_cos, full_sin, 4, 128), ops.rope_qkv_(qkv.clone(), full_cos,
                                                                                           full_sin, 4))
    a, m = torch.randn(2, 8, 32, generator=g), torch.randn(2, 8, 48, generator=g)
    wd, w4, bd, b4 = torch.randn(16, 32, generator=g), torch.randn(16, 48, generator=g), torch.randn(16), torch.randn(16)
    torch.testing.assert_close(ops.parallel_out(a, m, wd, w4, bd, b4), F.linear(a, wd, bd) + F.linear(m, w4, b4))


# ---------------------------------------------------------------------------------------------------------------
# the model against transformers
# ---------------------------------------------------------------------------------------------------------------
def _hf_config(cfg, transformers):
    d = {k: v for k, v in to_hf_config_dict(cfg).items() if k not in ("model_type", "architectures", "torch_dtype")}
    return transformers.GPTNeoXConfig(**d)


def _hf_neox(cfg, transformers):
    hf_cfg = _hf_config(cfg, transformers)
    hf_cfg._attn_implementation = "eager"
    return transformers.GPTNeoXForCausalLM(hf_cfg).float().eval()


def _spread(cfg):
    """fp32 model whose norm gains and every bias are away from their initial 1 and 0, so each is visible."""
    torch.manual_seed(0)
    mine = build_model(cfg, dtype=torch.float32, device="cpu")
    g = torch.Generator().manual_seed(3)
    with torch.no_grad():
        for n, p in mine.named_parameters():
            if "norm" in n and n.endswith("weight"):
                p.copy_(1 + 0.3 * torch.randn(p.shape, generator=g))
            elif n.endswith("bias"):
                p.copy_(0.1 * torch.randn(p.shape, generator=g))
    return mine


@pytest.mark.parametrize("name", DEBUG)
@pytest.mark.parametrize("tied", [False, True])
def test_debug_gpt_neox_matches_transformers_fp32(name, tied):
    transformers = pytest.importorskip("transformers")
    cfg = get_config(name, tie_word_embeddings=tied)
    assert cfg.arch == "gpt_neox" and cfg.parallel_residual and cfg.layer_norm and cfg.gelu_exact and cfg.all_bias
    assert cfg.rotary_dim == cfg.head_dim // 4 and cfg.rotary_dim < cfg.head_dim
    mine = _spread(cfg)
    hf = _hf_neox(cfg, transformers)
    assert hf.gpt_neox.layers[0].attention.rotary_ndims == cfg.rotary_dim
    hf.load_state_dict(gpt_neox_layout.to_hf_state_dict(mine.state_dict(), cfg.num_attention_heads), strict=True)
    ids = torch.randint(0, cfg.vocab_size, (2, 256), generator=torch.Generator().manual_seed(1))
    out_mine = mine(input_ids=ids, labels=ids, return_logits=True)
    out_hf = hf(input_ids=ids, labels=ids)
    assert torch.allclose(out_mine.logits, out_hf.logits, atol=2e-4, rtol=1e-3), \
        (out_mine.logits - out_hf.logits).abs().max()
    assert abs(out_mine.loss.item() - out_hf.loss.item()) < 1e-4
    # the partial rotation is in effect: rotating whole heads changes the logits
    whole = _spread(dataclasses.replace(cfg, partial_rotary_factor=1.0))
    assert (whole(input_ids=ids, return_logits=True).logits - out_mine.logits).abs().max() > 1e-3
    out_mine.loss.backward()
    out_hf.loss.backward()
    names = [n for n, _ in mine.named_parameters()]
    assert ("lm_head.weight" in names) == (not tied)
    hf_grads = {n: p.grad for n, p in hf.named_parameters()}
    if tied:
        hf_grads["embed_out.weight"] = hf_grads["gpt_neox.embed_in.weight"]
    want = gpt_neox_layout.from_hf_state_dict(hf_grads, names, cfg.num_attention_heads)
    for n, p in mine.named_parameters():
        err = ((p.grad - want[n]).norm() / want[n].norm()).item()
        assert err < 1e-4, (n, err)


def test_layout_round_trip_and_per_head_interleave():
    cfg = get_config("debug-gpt-neox-d64")
    sd = build_model(cfg, dtype=torch.float32, device="cpu").state_dict()
    hf = gpt_neox_layout.to_hf_state_dict(sd, cfg.num_attention_heads)
    nh, d, H = cfg.num_attention_heads, cfg.head_dim, cfg.hidden_size
    qkv = hf["gpt_neox.layers.1.attention.query_key_value.weight"].view(nh, 3, d, H)
    assert torch.equal(qkv[2, 1], sd["model.layers.1.self_attn.k_proj.weight"][2 * d:3 * d])   # head 2's k rows
    assert hf["gpt_neox.layers.0.attention.dense.bias"] is sd["model.layers.0.self_attn.o_proj.bias"]
    assert set(hf) >= {"gpt_neox.embed_in.weight", "embed_out.weight", "gpt_neox.final_layer_norm.bias",
                       "gpt_neox.layers.0.mlp.dense_h_to_4h.weight", "gpt_neox.layers.0.mlp.dense_4h_to_h.bias"}
    back = gpt_neox_layout.from_hf_state_dict(hf, list(sd), nh)
    assert all(torch.equal(back[k], v) for k, v in sd.items())
    with pytest.raises(KeyError):
        gpt_neox_layout.hf_name("model.layers.0.mlp.gate_proj.weight")


# ---------------------------------------------------------------------------------------------------------------
# configs
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("size", list(PYTHIA))
@pytest.mark.parametrize("suffix", ["", "-deduped"])
def test_registry_pythia(size, suffix):
    h, i, l, nh, v, n = PYTHIA[size]
    cfg = get_config(f"EleutherAI/pythia-{size}{suffix}")
    assert cfg.arch == "gpt_neox" and (cfg.vocab_size, cfg.hidden_size, cfg.intermediate_size) == (v, h, i)
    assert (cfg.num_hidden_layers, cfg.num_attention_heads, cfg.num_key_value_heads) == (l, nh, nh)
    assert cfg.head_dim in (64, 128) and cfg.rotary_dim == cfg.head_dim // 4 and not cfg.tie_word_embeddings
    assert (cfg.rope_theta, cfg.max_position_embeddings, cfg.layer_norm_epsilon) == (1e4, 2048, 1e-5)
    assert cfg.num_parameters() == n
    assert build_model(cfg, dtype=torch.bfloat16, device="meta").num_parameters() == n


def test_num_parameters_match_transformers_on_meta():
    transformers = pytest.importorskip("transformers")
    for name in [f"EleutherAI/pythia-{s}" for s in PYTHIA] + DEBUG:
        c = get_config(name)
        for tied in (True, False):
            c2 = dataclasses.replace(c, tie_word_embeddings=tied)
            with torch.device("meta"):
                hf = transformers.GPTNeoXForCausalLM(_hf_config(c2, transformers))
            assert sum(p.numel() for p in hf.parameters()) == c2.num_parameters(), (name, tied)
            assert build_model(c2, dtype=torch.bfloat16, device="meta").num_parameters() == c2.num_parameters()


def test_existing_configs_unchanged():
    assert get_config("meta-llama/Llama-2-7b-hf").num_parameters() == 6_738_415_616
    assert get_config("bigcode/starcoder2-3b").num_parameters() == 3_030_371_328
    for name in ("meta-llama/Llama-2-7b-hf", "bigcode/starcoder2-7b", "Qwen/Qwen3-8B", "debug-llama-d64"):
        c = get_config(name)
        assert c.partial_rotary_factor == 1.0 and c.rotary_dim == c.head_dim and not c.parallel_residual
    sc = get_config("debug-starcoder2")
    assert sc.gelu_mlp and not sc.gelu_exact


def _write_config(tmp_path, d):
    (tmp_path / "config.json").write_text(json.dumps(d))
    return str(tmp_path)


@pytest.mark.parametrize("name", DEBUG + ["EleutherAI/pythia-1.4b", "EleutherAI/pythia-410m-deduped"])
def test_hf_config_round_trip(tmp_path, name):
    cfg = get_config(name)
    d = to_hf_config_dict(cfg)
    assert d["model_type"] == "gpt_neox" and d["architectures"] == ["GPTNeoXForCausalLM"]
    assert d["use_parallel_residual"] and d["hidden_act"] == "gelu" and d["rotary_pct"] == 0.25
    back = get_config(_write_config(tmp_path, d))
    assert back.to_dict() == {**cfg.to_dict(), "name": str(tmp_path)}
    transformers = pytest.importorskip("transformers")
    hf = _hf_config(cfg, transformers)
    assert hf.rope_parameters["partial_rotary_factor"] == 0.25 and hf.rope_parameters["rope_theta"] == cfg.rope_theta
    assert hf.layer_norm_eps == cfg.layer_norm_epsilon and hf.use_parallel_residual and hf.attention_bias
    assert hf.tie_word_embeddings == cfg.tie_word_embeddings


def test_hf_config_layouts_and_refusals(tmp_path):
    d = to_hf_config_dict(get_config("debug-gpt-neox"))
    v5 = {k: v for k, v in d.items() if k not in ("rotary_pct", "rotary_emb_base")}   # transformers>=5
    v5["rope_parameters"] = {"rope_theta": 5e5, "rope_type": "default", "partial_rotary_factor": 0.5}
    cfg = get_config(_write_config(tmp_path, v5))
    assert (cfg.rope_theta, cfg.partial_rotary_factor, cfg.rotary_dim, cfg.arch) == (5e5, 0.5, 64, "gpt_neox")
    transformers = pytest.importorskip("transformers")
    saved = transformers.GPTNeoXConfig(**{k: v for k, v in d.items() if k not in ("model_type", "architectures")})
    saved.save_pretrained(str(tmp_path / "hf"))   # what transformers 5 writes
    assert get_config(str(tmp_path / "hf")).to_dict() == {**get_config("debug-gpt-neox").to_dict(),
                                                          "name": str(tmp_path / "hf")}
    assert get_config(_write_config(tmp_path, {**d, "rotary_pct": 1.0})).rotary_dim == 128
    assert get_config(_write_config(tmp_path, {**d, "layer_norm_eps": 1e-6})).layer_norm_epsilon == 1e-6
    for bad, key in (({"use_parallel_residual": False}, "use_parallel_residual"),
                     ({"hidden_act": "gelu_new"}, "hidden_act"),
                     ({"attention_bias": False}, "attention_bias"),
                     ({"hidden_dropout": 0.1}, "hidden_dropout"),
                     ({"attention_dropout": 0.1}, "attention_dropout"),
                     ({"rope_scaling": {"rope_type": "linear", "factor": 2.0}}, "rope_scaling"),
                     ({"rope_parameters": {"rope_theta": 1e4, "rope_type": "dynamic", "factor": 2.0}},
                      "rope_parameters"),
                     ({"num_attention_heads": 2}, "head_dim"),      # 512 / 2 = 256 (Pythia-1b)
                     ({"num_attention_heads": 32, "hidden_size": 2560}, "head_dim"),   # 80 (Pythia-2.8b)
                     ({"rotary_pct": 0.1}, "rotary_pct"),
                     ({"rope_parameters": {"rope_theta": 1e4, "partial_rotary_factor": 0.3}},
                      "partial_rotary_factor")):
        with pytest.raises(ValueError, match=key):
            get_config(_write_config(tmp_path, {**d, **bad}))
    with pytest.raises(ValueError, match="to 0.0"):
        get_config(_write_config(tmp_path, {**d, "hidden_dropout": 0.1}))


# ---------------------------------------------------------------------------------------------------------------
# --pretrained and the consolidation tool
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tied", [False, True])
def test_pretrained_hf_gpt_neox_checkpoint_loads(tmp_path, tied):
    transformers = pytest.importorskip("transformers")
    pytest.importorskip("safetensors")
    from distributed_training_guide_b200.tools.load_hf import maybe_load_pretrained

    cfg = get_config("debug-gpt-neox", tie_word_embeddings=tied)
    torch.manual_seed(5)
    hf = _hf_neox(cfg, transformers)
    with torch.no_grad():   # gains and biases away from 1 and 0, so that loading them is visible
        for n, p in hf.named_parameters():
            if "norm" in n or n.endswith("bias"):
                p.uniform_(0.5, 2.0)
    hf.save_pretrained(str(tmp_path / "m"), safe_serialization=True)
    loaded_cfg = get_config(str(tmp_path / "m"))
    assert loaded_cfg.arch == "gpt_neox" and loaded_cfg.tie_word_embeddings == tied
    assert loaded_cfg.rotary_dim == 32
    model = build_model(loaded_cfg, dtype=torch.float32, device="cpu")
    assert maybe_load_pretrained(SimpleNamespace(model_name=str(tmp_path / "m"), pretrained="require"), model=model)
    want = gpt_neox_layout.to_hf_state_dict(model.state_dict(), cfg.num_attention_heads)
    for k, v in hf.state_dict().items():
        assert torch.equal(want[k], v), k
    ids = torch.randint(0, cfg.vocab_size, (1, 64), generator=torch.Generator().manual_seed(2))
    with torch.no_grad():
        assert torch.allclose(model(input_ids=ids, return_logits=True).logits, hf(input_ids=ids).logits,
                              atol=2e-4, rtol=1e-3)


def _fsdp_load(rank, world):
    from distributed_training_guide_b200.engine import TrainEngine
    from distributed_training_guide_b200.tools.load_hf import load_into_fsdp

    eng = TrainEngine.create("debug-gpt-neox", parallelism="fsdp", batch_size=1, seq_length=64, device="cpu",
                             lr=1e-3, seed=5)
    cfg = get_config("debug-gpt-neox")
    src = build_model(cfg, dtype=torch.bfloat16, device="cpu")
    src.init_weights(seed=999)
    with torch.no_grad():
        for n, p in src.named_parameters():
            if n.endswith("bias"):
                p.uniform_(-1.0, 1.0)
    sd = src.state_dict()
    hf_sd = gpt_neox_layout.to_hf_state_dict(sd, cfg.num_attention_heads)   # as a GPT-NeoX checkpoint holds it
    reader = gpt_neox_layout.HFReader(hf_sd.__getitem__, hf_sd.keys(), cfg.num_attention_heads)
    load_into_fsdp(eng.strategy.engine, reader if rank == 0 else None)
    full = eng.strategy.engine.full_state_dict()
    return all(torch.equal(v.to(sd[k].dtype), sd[k]) for k, v in full.items()), set(full) == set(sd)


def test_fsdp_pretrained_load_covers_every_parameter():
    res = run_distributed(_fsdp_load, world=2, args=(), timeout=600)
    assert all(r == (True, True) for r in res), res


def test_chapter04_checkpoint_consolidates_to_a_strict_gpt_neox_state_dict(tmp_path):
    transformers = pytest.importorskip("transformers")
    root = Path(__file__).resolve().parent.parent
    script = root / "04-fully-sharded-data-parallel" / "train_llm.py"
    cmd = [sys.executable, "-m", "torch.distributed.run", "--standalone", "--local-addr", "127.0.0.1",
           "--nproc-per-node", "2", str(script), "-d", "synthetic", "-m", "debug-gpt-neox", "-s", "128", "-b", "1",
           "--num-samples", "16", "--log-freq", "1", "--device", "cpu", "--save-dir", str(tmp_path), "-e", "exp",
           "--ckpt-freq", "2", "--lr", "1e-3", "--max-steps", "2"]
    r = subprocess.run(cmd, capture_output=True, text=True, cwd=str(script.parent), timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    from distributed_training_guide_b200.tools.consolidate import consolidate

    sd = torch.load(consolidate(str(tmp_path / "exp"), "debug-gpt-neox", world=2), weights_only=True)
    hf = _hf_neox(get_config("debug-gpt-neox"), transformers)
    for k in ("gpt_neox.layers.1.mlp.dense_4h_to_h.bias", "gpt_neox.final_layer_norm.bias",
              "gpt_neox.layers.0.attention.dense.bias", "gpt_neox.layers.0.attention.query_key_value.bias"):
        assert sd[k].abs().sum() > 0, k   # trained away from their zero init
    hf.load_state_dict({k: v.float() for k, v in sd.items()}, strict=True)


# ---------------------------------------------------------------------------------------------------------------
# flat layout and the layer
# ---------------------------------------------------------------------------------------------------------------
def test_flat_order_holds_every_parameter_with_the_matrices_first():
    from distributed_training_guide_b200.models.llama import LayerNorm, Starcoder2MLP
    from distributed_training_guide_b200.parallel.flat import build_groups

    model = build_model(get_config("debug-gpt-neox"), dtype=torch.bfloat16, device="cpu")
    layer = model.model.layers[0]
    # StarCoder2's parameters with the parallel residual and the exact GELU
    assert isinstance(layer.input_layernorm, LayerNorm) and isinstance(layer.post_attention_layernorm, LayerNorm)
    assert isinstance(layer.mlp, Starcoder2MLP) and layer.gelu_exact
    assert layer.parallel_residual and not layer.post_norm
    order = layer.flat_order
    assert order == ("self_attn.q_proj.weight", "self_attn.k_proj.weight", "self_attn.v_proj.weight",
                     "self_attn.o_proj.weight", "mlp.c_fc.weight", "mlp.c_proj.weight", "input_layernorm.weight",
                     "input_layernorm.bias", "post_attention_layernorm.weight", "post_attention_layernorm.bias",
                     "self_attn.q_proj.bias", "self_attn.k_proj.bias", "self_attn.v_proj.bias",
                     "self_attn.o_proj.bias", "mlp.c_fc.bias", "mlp.c_proj.bias")
    assert layer.fused == {"qkv": order[:3], "qkv_bias": order[10:13]}
    assert set(order) == {n for n, _ in layer.named_parameters()} and len(order) == len(set(order))
    named = dict(layer.named_parameters())
    dims = [named[n].dim() for n in order]
    assert dims == sorted(dims, reverse=True), "matrices first"
    assert all(named[n].numel() % 8 == 0 for n in order)
    groups = build_groups(model, "cpu", torch.bfloat16)
    assert len({id(p) for g in groups for p in g.params}) == len(list(model.parameters()))
    assert set(layer._fused) == {"qkv", "qkv_bias"}
    assert layer._fused["qkv"].data.shape == (3 * 512, 512) and layer._fused["qkv_bias"].data.shape == (3 * 512,)


@pytest.mark.parametrize("name", DEBUG)
def test_layer_equals_the_reference_parallel_residual(name):
    """Each layer's (branch, h) against the ops' reference math, with HF's ``(m + a) + h`` as the next stream."""
    cfg = get_config(name)
    model = _spread(cfg)
    S, nh, d, rot = 32, cfg.num_attention_heads, cfg.head_dim, cfg.rotary_dim
    ids = torch.randint(0, cfg.vocab_size, (1, S), generator=torch.Generator().manual_seed(4))
    m = model.model
    cos, sin = m.rotary_emb.tables(S, ids.device)
    assert cos.shape == (S, rot // 2)
    x, res = m.embed_tokens(ids), None
    stream = x
    for layer in m.layers:
        out, h = layer(x, res, cos, sin)
        att, mlp, eps = layer.self_attn, layer.mlp, cfg.layer_norm_epsilon
        n1, n2 = layer.input_layernorm, layer.post_attention_layernorm
        y1 = ref.layer_norm(stream, n1.weight, n1.bias, eps)
        y2 = ref.layer_norm(stream, n2.weight, n2.bias, eps)
        q = ref.linear(y1, att.q_proj.weight, att.q_proj.bias).view(1, S, nh, d)
        k = ref.linear(y1, att.k_proj.weight, att.k_proj.bias).view(1, S, nh, d)
        v = ref.linear(y1, att.v_proj.weight, att.v_proj.bias).view(1, S, nh, d)
        q = torch.cat([ref.rope_apply(q[..., :rot], cos, sin), q[..., rot:]], dim=-1)
        k = torch.cat([ref.rope_apply(k[..., :rot], cos, sin), k[..., rot:]], dim=-1)
        a = ref.linear(ref.attention(q, k, v).reshape(1, S, nh * d), att.o_proj.weight, att.o_proj.bias)
        mo = ref.linear(F.gelu(ref.linear(y2, mlp.c_fc.weight, mlp.c_fc.bias)), mlp.c_proj.weight, mlp.c_proj.bias)
        torch.testing.assert_close(h, stream)
        torch.testing.assert_close(out, a + mo)
        new_stream = (mo + a) + stream   # HF: hidden_states = mlp_output + attn_output + hidden_states
        torch.testing.assert_close(out + h, new_stream)
        x, res, stream = out, h, new_stream


# ---------------------------------------------------------------------------------------------------------------
# engines over gloo against one process
# ---------------------------------------------------------------------------------------------------------------
S_DIST, LR_DIST, B_GLOBAL = 256, 5e-3, 4


def _batch(vocab, step, rank, B=1):
    g = torch.Generator().manual_seed(1000 * step + rank)
    ids = torch.randint(0, vocab, (B, S_DIST), generator=g)
    return {"input_ids": ids, "labels": ids.clone()}


def _tail(model):
    """Every norm gain and bias and every projection bias, per layer, then the final norm's."""
    out = [torch.cat([p.detach().float().reshape(-1) for n, p in l.named_parameters() if p.dim() == 1])
           for l in model.model.layers]
    out.append(torch.cat([model.model.norm.weight.detach().float(), model.model.norm.bias.detach().float()]))
    return out


def _train_dist(rank, world, parallelism, steps):
    from distributed_training_guide_b200.engine import TrainEngine

    torch.manual_seed(0)
    per = B_GLOBAL // world
    eng = TrainEngine.create("debug-gpt-neox", parallelism=parallelism, batch_size=per, seq_length=S_DIST,
                             device="cpu", lr=LR_DIST)
    dp_rank = eng.strategy.dp_rank
    losses, tails = [], []
    for i in range(steps):
        parts = [_batch(eng.config.vocab_size, i, dp_rank * per + j) for j in range(per)]
        losses.append(float(eng.step({k: torch.cat([p[k] for p in parts]) for k in parts[0]})))
        if parallelism != "fsdp":
            tails.append(_tail(eng.model))
    if parallelism == "fsdp":
        full = eng.strategy.engine.full_state_dict()
        tails.append([full["model.norm.bias"].float(), full["model.layers.1.mlp.c_proj.bias"].float()])
    return losses, tails, eng.strategy.dp_size


def _single(steps):
    from distributed_training_guide_b200.engine import TrainEngine

    torch.manual_seed(0)
    eng = TrainEngine.create("debug-gpt-neox", parallelism="single", batch_size=B_GLOBAL, seq_length=S_DIST,
                             device="cpu", lr=LR_DIST)
    losses, tails = [], []
    for i in range(steps):
        parts = [_batch(eng.config.vocab_size, i, r) for r in range(B_GLOBAL)]
        losses.append(float(eng.step({k: torch.cat([p[k] for p in parts]) for k in parts[0]})))
        tails.append(_tail(eng.model))
    sd = eng.model.state_dict()
    return losses, tails, [sd["model.norm.bias"].float(), sd["model.layers.1.mlp.c_proj.bias"].float()]


@pytest.mark.parametrize("parallelism", ["ddp", "fsdp"])
def test_distributed_gpt_neox_matches_single_process(parallelism):
    steps, world = 3, 2
    res = run_distributed(_train_dist, world=world, args=(parallelism, steps), timeout=600)
    assert res[0][2] == world
    ref_losses, ref_tails, ref_final = _single(steps)
    for i in range(steps):
        mean = float(np.mean([r[0][i] for r in res]))
        assert abs(mean - ref_losses[i]) < 2e-2, (parallelism, i, [r[0][i] for r in res], ref_losses[i])
    if parallelism == "fsdp":
        for j, want in enumerate(ref_final):
            a, want = np.asarray(res[0][1][0][j]), want.numpy()
            assert np.array_equal(a, np.asarray(res[1][1][0][j])), "differs between ranks"
            assert np.abs(a - want).max() <= 2 * 2.0 ** -7, np.abs(a - want).max()
            assert np.abs(a).sum() > 0
        return
    for i in range(steps):
        for layer in range(len(ref_tails[i])):
            a, b = res[0][1][i][layer], res[1][1][i][layer]
            assert np.array_equal(a, b), (parallelism, i, layer, "differs between ranks")
            want = ref_tails[i][layer].numpy()
            assert np.abs(a - want).max() <= 2 * 2.0 ** -7, (parallelism, i, layer, np.abs(a - want).max())


@pytest.mark.parametrize("flags", [dict(fp8=True), dict(max_grad_norm=1.0), dict(checkpoint_activations=True),
                                   dict(document_masking=True)])
def test_single_engine_flags_train_gpt_neox(flags):
    """The flags a Llama run takes also train debug-gpt-neox: finite losses, and every bias and gain moves."""
    from distributed_training_guide_b200.engine import TrainEngine

    torch.manual_seed(0)
    eng = TrainEngine.create("debug-gpt-neox", parallelism="single", batch_size=1, seq_length=128, device="cpu",
                             lr=LR_DIST, **flags)
    t0 = _tail(eng.model)
    for i in range(2):
        b = _batch(eng.config.vocab_size, i, 0)
        b = {k: v[:, :128] for k, v in b.items()}
        if flags.get("document_masking"):
            b["position_ids"] = torch.cat([torch.arange(50), torch.arange(78)])[None]
        assert math.isfinite(float(eng.step(b)))
    assert all(not torch.equal(a, b) for a, b in zip(t0, _tail(eng.model)))


def test_gradient_accumulation_matches_the_unaccumulated_step():
    from distributed_training_guide_b200.parallel.flat import build_groups

    cfg = get_config("debug-gpt-neox")
    model = _spread(cfg)
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
    assert ((acc - full).norm() / full.norm()).item() < 1e-5


@pytest.mark.parametrize("parallelism", ["tp", "2d"])
def test_tensor_parallel_engines_refuse_gpt_neox(parallelism):
    from distributed_training_guide_b200.engine import TrainEngine

    with pytest.raises(ValueError, match="parallel residual") as e:
        TrainEngine.create("debug-gpt-neox", parallelism=parallelism, batch_size=1, seq_length=128, device="cpu",
                           tensor_parallel=1)
    assert "single-GPU, DDP or FSDP" in str(e.value)
