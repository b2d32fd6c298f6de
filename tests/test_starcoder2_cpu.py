"""StarCoder2 on the CPU: ``debug-starcoder2`` against ``transformers.Starcoder2ForCausalLM`` with the same weights
(logits, loss and every gradient; tied, untied and with a window shorter than the sequence), the new ops' CPU paths,
the registry's parameter counts against the meta-device models, the HF config round trip and its refusals, an HF
checkpoint loaded through ``--pretrained`` and written back by the consolidation tool, the layer's flat layout, DDP /
FSDP over gloo against one process, the single-engine flags, and the refusal of the tensor-parallel engines."""
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
from distributed_training_guide_b200.models import build_model, get_config, to_hf_config_dict
from distributed_training_guide_b200.ops import reference as ref

STARCODER2 = {   # id: (hidden, intermediate, layers, heads, kv heads, rope theta, tied, parameters)
    "bigcode/starcoder2-3b": (3072, 12288, 30, 24, 2, 999999.4420358813, True, 3_030_371_328),
    "bigcode/starcoder2-7b": (4608, 18432, 32, 36, 4, 1e6, True, 7_173_923_840),
    "bigcode/starcoder2-15b": (6144, 24576, 40, 48, 4, 1e5, False, 15_957_889_024),
}


# ---------------------------------------------------------------------------------------------------------------
# the ops' CPU paths
# ---------------------------------------------------------------------------------------------------------------
def test_layer_norm_and_gelu_cpu_paths():
    g = torch.Generator().manual_seed(0)
    x = (torch.randn(16, 64, generator=g) * 3 + 1).bfloat16()
    r = torch.randn(16, 64, generator=g).bfloat16()
    w, b = (torch.randn(64, generator=g)).bfloat16(), torch.randn(64, generator=g).bfloat16()
    y = ops.layer_norm(x, w, b, 1e-5)
    assert y.dtype == torch.bfloat16 and torch.equal(y, ref.layer_norm(x, w, b, 1e-5))
    xf = x.double()
    y64 = (xf - xf.mean(-1, keepdim=True)) / torch.sqrt(xf.var(-1, unbiased=False, keepdim=True) + 1e-5)
    y64 = y64 * w.double() + b.double()
    assert ((y.double() - y64).abs() <= y64.abs() * 2.0 ** -8 + 1e-5).all()   # one rounding
    y2, h = ops.add_layer_norm(x, r, w, b, 1e-5)
    assert torch.equal(h, x + r) and torch.equal(y2, ref.layer_norm(x + r, w, b, 1e-5))
    t = torch.linspace(-8, 8, 4096)
    torch.testing.assert_close(ops.gelu_tanh(t), F.gelu(t, approximate="tanh"), rtol=1e-6, atol=1e-6)
    assert torch.equal(ops.gelu_tanh(t.bfloat16()), ref.gelu_new(t.bfloat16().float()).bfloat16())


# ---------------------------------------------------------------------------------------------------------------
# the model against transformers
# ---------------------------------------------------------------------------------------------------------------
def _hf_starcoder2(cfg, transformers):
    d = {k: v for k, v in to_hf_config_dict(cfg).items() if k not in ("model_type", "architectures", "torch_dtype")}
    hf_cfg = transformers.Starcoder2Config(**d)
    hf_cfg._attn_implementation = "eager"
    return transformers.Starcoder2ForCausalLM(hf_cfg).float().eval()


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


@pytest.mark.parametrize("tied,window", [(True, None), (False, None), (True, 192)])
def test_debug_starcoder2_matches_transformers_fp32(tied, window):
    transformers = pytest.importorskip("transformers")
    cfg = get_config("debug-starcoder2", tie_word_embeddings=tied)
    if window is not None:
        cfg = dataclasses.replace(cfg, sliding_window=window)
    assert cfg.arch == "starcoder2" and cfg.layer_norm and cfg.gelu_mlp and cfg.all_bias and cfg.head_dim == 128
    mine = _spread(cfg)
    hf = _hf_starcoder2(cfg, transformers)
    missing, unexpected = hf.load_state_dict(mine.state_dict(), strict=False)
    assert not unexpected, unexpected
    assert all("rotary" in m or "inv_freq" in m for m in missing), missing   # names are HF's
    assert [n for n, _ in mine.named_parameters()] == [n for n, _ in hf.named_parameters()]   # and so is the order
    ids = torch.randint(0, cfg.vocab_size, (2, 256), generator=torch.Generator().manual_seed(1))
    out_mine = mine(input_ids=ids, labels=ids, return_logits=True)
    out_hf = hf(input_ids=ids, labels=ids)
    assert torch.allclose(out_mine.logits, out_hf.logits, atol=2e-4, rtol=1e-3), \
        (out_mine.logits - out_hf.logits).abs().max()
    assert abs(out_mine.loss.item() - out_hf.loss.item()) < 1e-4
    if window is not None:   # the window is in effect: without it the logits differ
        full = _spread(dataclasses.replace(cfg, sliding_window=None))
        assert (full(input_ids=ids, return_logits=True).logits - out_mine.logits).abs().max() > 1e-3
    out_mine.loss.backward()
    out_hf.loss.backward()
    hf_params = dict(hf.named_parameters())
    names = [n for n, _ in mine.named_parameters()]
    for key in ("o_proj.bias", "c_fc.bias", "c_proj.bias", "q_proj.bias", "input_layernorm.bias", "model.norm.bias"):
        assert any(n.endswith(key) for n in names), key
    assert ("lm_head.weight" in names) == (not tied)
    for n, p in mine.named_parameters():
        want = hf_params[n].grad
        err = ((p.grad - want).norm() / want.norm()).item()
        assert err < 1e-4, (n, err)


# ---------------------------------------------------------------------------------------------------------------
# configs
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(STARCODER2))
def test_registry_starcoder2(name):
    h, i, l, nh, nkv, theta, tied, n = STARCODER2[name]
    cfg = get_config(name)
    assert cfg.arch == "starcoder2" and cfg.head_dim == 128 and not cfg.qkv_bias and not cfg.qk_norm
    assert (cfg.vocab_size, cfg.hidden_size, cfg.intermediate_size, cfg.num_hidden_layers) == (49152, h, i, l)
    assert (cfg.num_attention_heads, cfg.num_key_value_heads, cfg.tie_word_embeddings) == (nh, nkv, tied)
    assert (cfg.rope_theta, cfg.layer_norm_epsilon, cfg.max_position_embeddings) == (theta, 1e-5, 16384)
    assert cfg.sliding_window == 4096
    assert cfg.num_parameters() == n
    assert build_model(cfg, dtype=torch.bfloat16, device="meta").num_parameters() == n


def test_num_parameters_meta_and_transformers():
    cfg = get_config("debug-starcoder2")
    assert build_model(cfg, dtype=torch.float32, device="meta").num_parameters() == cfg.num_parameters()
    transformers = pytest.importorskip("transformers")
    for name in list(STARCODER2) + ["debug-starcoder2"]:
        c = get_config(name)
        for tied in (True, False):
            c2 = dataclasses.replace(c, tie_word_embeddings=tied)
            d = {k: v for k, v in to_hf_config_dict(c2).items()
                 if k not in ("model_type", "architectures", "torch_dtype")}
            with torch.device("meta"):
                hf = transformers.Starcoder2ForCausalLM(transformers.Starcoder2Config(**d))
            assert sum(p.numel() for p in hf.parameters()) == c2.num_parameters(), (name, tied)


def test_existing_parameter_counts_unchanged():
    assert get_config("meta-llama/Llama-2-7b-hf").num_parameters() == 6_738_415_616
    assert get_config("allenai/OLMo-2-1124-7B").num_parameters() == 7_298_617_344


def _write_config(tmp_path, d):
    (tmp_path / "config.json").write_text(json.dumps(d))
    return str(tmp_path)


@pytest.mark.parametrize("name", list(STARCODER2) + ["debug-starcoder2"])
def test_hf_config_round_trip(tmp_path, name):
    cfg = get_config(name)
    d = to_hf_config_dict(cfg)
    assert d["model_type"] == "starcoder2" and d["architectures"] == ["Starcoder2ForCausalLM"]
    assert d["attention_dropout"] == d["residual_dropout"] == d["embedding_dropout"] == 0.0
    back = get_config(_write_config(tmp_path, d))
    assert back.to_dict() == {**cfg.to_dict(), "name": str(tmp_path)}
    transformers = pytest.importorskip("transformers")
    hf = transformers.Starcoder2Config(**{k: v for k, v in d.items() if k not in ("model_type", "architectures")})
    assert hf.num_key_value_heads == cfg.num_key_value_heads and hf.tie_word_embeddings == cfg.tie_word_embeddings
    assert hf.rope_parameters["rope_theta"] == cfg.rope_theta and hf.norm_epsilon == cfg.layer_norm_epsilon
    assert hf.sliding_window == cfg.sliding_window and hf.use_bias


def test_hf_config_layouts_and_refusals(tmp_path):
    d = to_hf_config_dict(get_config("debug-starcoder2"))
    v5 = {k: v for k, v in d.items() if k != "rope_theta"}   # transformers>=5 writes rope_parameters
    v5["rope_parameters"] = {"rope_theta": 5e5, "rope_type": "default"}
    cfg = get_config(_write_config(tmp_path, v5))
    assert cfg.rope_theta == 5e5 and cfg.rope_scaling is None and cfg.arch == "starcoder2"
    assert get_config(_write_config(tmp_path, {**d, "sliding_window": None})).sliding_window is None
    assert get_config(_write_config(tmp_path, {**d, "norm_epsilon": 1e-6})).layer_norm_epsilon == 1e-6
    assert get_config(_write_config(tmp_path, {**d, "tie_word_embeddings": False})).tie_word_embeddings is False
    # the older payloads' keys, at their supported values
    assert get_config(_write_config(tmp_path, {**d, "norm_type": "layer_norm", "mlp_type": "default"})).layer_norm
    for bad, key in (({"use_bias": False}, "use_bias"),
                     ({"hidden_act": "gelu"}, "hidden_act"),
                     ({"norm_type": "rms_norm"}, "norm_type"),
                     ({"mlp_type": "gated"}, "mlp_type"),
                     ({"rope_parameters": {"rope_theta": 1e5, "rope_type": "yarn", "factor": 4.0}}, "rope_parameters"),
                     ({"rope_scaling": {"rope_type": "linear", "factor": 2.0}}, "rope_scaling"),
                     ({"head_dim": 64}, "head_dim"),
                     ({"attention_dropout": 0.1}, "attention_dropout"),
                     ({"residual_dropout": 0.1}, "residual_dropout"),
                     ({"embedding_dropout": 0.1}, "embedding_dropout")):
        with pytest.raises(ValueError, match=key):
            get_config(_write_config(tmp_path, {**d, **bad}))
    with pytest.raises(ValueError, match="to 0.0"):
        get_config(_write_config(tmp_path, {**d, "residual_dropout": 0.1}))
    assert get_config(_write_config(tmp_path, {**d, "head_dim": 128})).head_dim == 128


# ---------------------------------------------------------------------------------------------------------------
# --pretrained and the consolidation tool
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tied", [True, False])
def test_pretrained_hf_starcoder2_checkpoint_loads(tmp_path, tied):
    transformers = pytest.importorskip("transformers")
    pytest.importorskip("safetensors")
    from distributed_training_guide_b200.tools.load_hf import maybe_load_pretrained

    cfg = get_config("debug-starcoder2", tie_word_embeddings=tied)
    torch.manual_seed(5)
    hf = _hf_starcoder2(cfg, transformers)
    with torch.no_grad():   # gains and biases away from 1 and 0, so that loading them is visible
        for n, p in hf.named_parameters():
            if "norm" in n or n.endswith("bias"):
                p.uniform_(0.5, 2.0)
    hf.save_pretrained(str(tmp_path / "m"), safe_serialization=True)
    loaded_cfg = get_config(str(tmp_path / "m"))
    assert loaded_cfg.arch == "starcoder2" and loaded_cfg.tie_word_embeddings == tied
    model = build_model(loaded_cfg, dtype=torch.float32, device="cpu")
    assert maybe_load_pretrained(SimpleNamespace(model_name=str(tmp_path / "m"), pretrained="require"), model=model)
    hf_sd = hf.state_dict()
    for k, v in model.state_dict().items():
        assert torch.equal(v, hf_sd[k]), k
    ids = torch.randint(0, cfg.vocab_size, (1, 64), generator=torch.Generator().manual_seed(2))
    with torch.no_grad():
        assert torch.allclose(model(input_ids=ids, return_logits=True).logits, hf(input_ids=ids).logits,
                              atol=2e-4, rtol=1e-3)


def _fsdp_load(rank, world):
    from distributed_training_guide_b200.engine import TrainEngine
    from distributed_training_guide_b200.tools.load_hf import load_into_fsdp

    eng = TrainEngine.create("debug-starcoder2", parallelism="fsdp", batch_size=1, seq_length=64, device="cpu",
                             lr=1e-3, seed=5)
    src = build_model(get_config("debug-starcoder2"), dtype=torch.bfloat16, device="cpu")
    src.init_weights(seed=999)
    with torch.no_grad():
        for n, p in src.named_parameters():
            if n.endswith("bias"):
                p.uniform_(-1.0, 1.0)
    sd = src.state_dict()
    load_into_fsdp(eng.strategy.engine, (lambda name: sd[name]) if rank == 0 else None)
    full = eng.strategy.engine.full_state_dict()
    # tied: the lm_head is the embedding, held once
    return all(torch.equal(v.to(sd[k].dtype), sd[k]) for k, v in full.items()), set(full) == set(sd) - {"lm_head.weight"}


def test_fsdp_pretrained_load_covers_every_parameter():
    res = run_distributed(_fsdp_load, world=2, args=(), timeout=600)
    assert all(r == (True, True) for r in res), res


def test_chapter04_checkpoint_consolidates_to_hf_names(tmp_path):
    transformers = pytest.importorskip("transformers")
    root = Path(__file__).resolve().parent.parent
    script = root / "04-fully-sharded-data-parallel" / "train_llm.py"
    cmd = [sys.executable, "-m", "torch.distributed.run", "--standalone", "--local-addr", "127.0.0.1",
           "--nproc-per-node", "2", str(script), "-d", "synthetic", "-m", "debug-starcoder2", "-s", "128", "-b", "1",
           "--num-samples", "16", "--log-freq", "1", "--device", "cpu", "--save-dir", str(tmp_path), "-e", "exp",
           "--ckpt-freq", "2", "--lr", "1e-3", "--max-steps", "2"]
    r = subprocess.run(cmd, capture_output=True, text=True, cwd=str(script.parent), timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    from distributed_training_guide_b200.tools.consolidate import consolidate

    sd = torch.load(consolidate(str(tmp_path / "exp"), "debug-starcoder2", world=2), weights_only=True)
    cfg = get_config("debug-starcoder2")
    hf = _hf_starcoder2(cfg, transformers)
    want = hf.state_dict()
    assert set(want) - {"lm_head.weight"} <= set(sd), set(want) - set(sd)
    for k in ("model.layers.1.mlp.c_proj.bias", "model.norm.bias", "model.layers.0.self_attn.o_proj.bias"):
        assert sd[k].shape == want[k].shape and sd[k].abs().sum() > 0, k   # trained away from their zero init
    missing, unexpected = hf.load_state_dict({k: v.float() for k, v in sd.items()}, strict=False)
    assert not unexpected, unexpected


# ---------------------------------------------------------------------------------------------------------------
# flat layout
# ---------------------------------------------------------------------------------------------------------------
def test_flat_order_holds_every_parameter_with_the_matrices_first():
    from distributed_training_guide_b200.models.llama import LayerNorm, Starcoder2MLP
    from distributed_training_guide_b200.parallel.flat import build_groups

    model = build_model(get_config("debug-starcoder2"), dtype=torch.bfloat16, device="cpu")
    layer = model.model.layers[0]
    # LayerNorms, the c_fc -> GELU-tanh -> c_proj MLP and the pre-norm residual with its add deferred
    assert isinstance(layer.input_layernorm, LayerNorm) and isinstance(layer.post_attention_layernorm, LayerNorm)
    assert isinstance(layer.mlp, Starcoder2MLP) and not layer.gelu_exact
    assert not layer.post_norm and not layer.parallel_residual
    order = layer.flat_order
    assert set(order) == {n for n, _ in layer.named_parameters()} and len(order) == len(set(order))
    named = dict(layer.named_parameters())
    dims = [named[n].dim() for n in order]
    assert dims == sorted(dims, reverse=True), "matrices first"
    assert order[:6] == ("self_attn.q_proj.weight", "self_attn.k_proj.weight", "self_attn.v_proj.weight",
                         "self_attn.o_proj.weight", "mlp.c_fc.weight", "mlp.c_proj.weight")
    assert order[6:10] == ("input_layernorm.weight", "input_layernorm.bias", "post_attention_layernorm.weight",
                           "post_attention_layernorm.bias")
    assert order[10:13] == ("self_attn.q_proj.bias", "self_attn.k_proj.bias", "self_attn.v_proj.bias")
    assert layer.fused == {"qkv": order[:3], "qkv_bias": order[10:13]}
    assert order[13:] == ("self_attn.o_proj.bias", "mlp.c_fc.bias", "mlp.c_proj.bias")
    assert all(named[n].numel() % 8 == 0 for n in order)
    groups = build_groups(model, "cpu", torch.bfloat16)
    assert len({id(p) for g in groups for p in g.params}) == len(list(model.parameters()))
    assert [n.split(".", 3)[-1] for n in groups[1].names] == list(order)
    assert set(layer._fused) == {"qkv", "qkv_bias"}   # no gate|up
    assert layer._fused["qkv"].data.shape == (512 + 2 * 256, 512)
    assert layer._fused["qkv_bias"].data.shape == (512 + 2 * 256,)
    # a parameter left out of the flat order is refused
    layer.flat_order = order[:-1]
    with pytest.raises(AssertionError, match="outside flat_order"):
        build_groups(model, "cpu", torch.bfloat16)
    llama = build_model(get_config("debug-llama-gqa"), dtype=torch.bfloat16, device="meta")
    assert llama.model.layers[0].flat_order == (
        "self_attn.q_proj.weight", "self_attn.k_proj.weight", "self_attn.v_proj.weight", "self_attn.o_proj.weight",
        "mlp.gate_proj.weight", "mlp.up_proj.weight", "mlp.down_proj.weight", "input_layernorm.weight",
        "post_attention_layernorm.weight")


def test_layer_equals_the_reference_ops_and_defers_the_add():
    cfg = dataclasses.replace(get_config("debug-starcoder2"), sliding_window=24)
    model = _spread(cfg)
    ids = torch.randint(0, cfg.vocab_size, (1, 32), generator=torch.Generator().manual_seed(4))
    m = model.model
    cos, sin = m.rotary_emb.tables(32, ids.device)
    x, res = m.embed_tokens(ids), None
    for layer in m.layers:
        out, h = layer(x, res, cos, sin)
        hh = x if res is None else x + res
        att, mlp, eps = layer.self_attn, layer.mlp, cfg.layer_norm_epsilon
        n1, n2 = layer.input_layernorm, layer.post_attention_layernorm
        y = ref.layer_norm(hh, n1.weight, n1.bias, eps)
        qkv = ref.linear(y, torch.cat([att.q_proj.weight, att.k_proj.weight, att.v_proj.weight]),
                         torch.cat([att.q_proj.bias, att.k_proj.bias, att.v_proj.bias])).view(1, 32, 8, 128)
        qkv = ref.rope_apply(qkv[:, :, :6], cos, sin)
        v = ref.linear(y, att.v_proj.weight, att.v_proj.bias).view(1, 32, 2, 128)
        a = ref.attention(qkv[:, :, :4], qkv[:, :, 4:6], v, window=24).reshape(1, 32, 512)
        h2 = ref.linear(a, att.o_proj.weight, att.o_proj.bias) + hh
        y2 = ref.layer_norm(h2, n2.weight, n2.bias, eps)
        want = ref.linear(ref.gelu_new(ref.linear(y2, mlp.c_fc.weight, mlp.c_fc.bias)), mlp.c_proj.weight,
                          mlp.c_proj.bias)
        torch.testing.assert_close(h, h2)
        torch.testing.assert_close(out, want)
        x, res = out, h


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
    eng = TrainEngine.create("debug-starcoder2", parallelism=parallelism, batch_size=per, seq_length=S_DIST,
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
    eng = TrainEngine.create("debug-starcoder2", parallelism="single", batch_size=B_GLOBAL, seq_length=S_DIST,
                             device="cpu", lr=LR_DIST)
    losses, tails = [], []
    for i in range(steps):
        parts = [_batch(eng.config.vocab_size, i, r) for r in range(B_GLOBAL)]
        losses.append(float(eng.step({k: torch.cat([p[k] for p in parts]) for k in parts[0]})))
        tails.append(_tail(eng.model))
    sd = eng.model.state_dict()
    return losses, tails, [sd["model.norm.bias"].float(), sd["model.layers.1.mlp.c_proj.bias"].float()]


@pytest.mark.parametrize("parallelism", ["ddp", "fsdp"])
def test_distributed_starcoder2_matches_single_process(parallelism):
    steps, world = 3, 2
    res = run_distributed(_train_dist, world=world, args=(parallelism, steps), timeout=600)
    assert res[0][2] == world
    ref_losses, ref_tails, ref_final = _single(steps)
    for i in range(steps):
        mean = float(np.mean([r[0][i] for r in res]))
        assert abs(mean - ref_losses[i]) < 2e-2, (parallelism, i, [r[0][i] for r in res], ref_losses[i])
    if parallelism == "fsdp":
        # the tail FSDP prefetches (norm gains and biases, every bias) was gathered and updated like one process's
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
            # bf16 tolerance: two ulps at magnitude 1 (gains), or the same absolute step for the biases near 0
            assert np.abs(a - want).max() <= 2 * 2.0 ** -7, (parallelism, i, layer, np.abs(a - want).max())


@pytest.mark.parametrize("flags", [dict(fp8=True), dict(max_grad_norm=1.0), dict(checkpoint_activations=True),
                                   dict(document_masking=True)])
def test_single_engine_flags_train_starcoder2(flags):
    """The flags a Llama run takes also train debug-starcoder2: finite losses, and every bias and gain moves."""
    from distributed_training_guide_b200.engine import TrainEngine

    torch.manual_seed(0)
    eng = TrainEngine.create("debug-starcoder2", parallelism="single", batch_size=1, seq_length=128, device="cpu",
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

    cfg = get_config("debug-starcoder2")
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
def test_tensor_parallel_engines_refuse_starcoder2(parallelism):
    from distributed_training_guide_b200.engine import TrainEngine

    with pytest.raises(ValueError, match="row-parallel o_proj / c_proj"):
        TrainEngine.create("debug-starcoder2", parallelism=parallelism, batch_size=1, seq_length=128, device="cpu",
                           tensor_parallel=1)


def _tp2(rank, world):
    from distributed_training_guide_b200.engine import TrainEngine

    try:
        TrainEngine.create("debug-starcoder2", parallelism="2d", batch_size=1, seq_length=256, device="cpu",
                           tensor_parallel=2)
    except ValueError as e:
        return str(e)
    return None


def test_two_rank_tensor_parallel_refuses_starcoder2():
    res = run_distributed(_tp2, world=2, args=(), timeout=300)
    assert all(r is not None and "row-parallel o_proj / c_proj" in r for r in res), res
