"""OLMoE on the CPU: the fp32 reference path against transformers' ``OlmoeForCausalLM`` (logits, loss and every
parameter's gradient, with the load-balancing loss off and on), the registry's parameter counts, reading and refusing
HF configs, the flat-buffer layout, and the refusals of tensor parallelism and fp8."""
import dataclasses
from types import SimpleNamespace

import pytest
import torch

from distributed_training_guide_b200.models.configs import _from_hf_dict, get_config, to_hf_config_dict
from distributed_training_guide_b200.models.llama import build_llama, decoder_layout
from distributed_training_guide_b200.ops import reference as ref

transformers = pytest.importorskip("transformers")
from transformers import OlmoeConfig, OlmoeForCausalLM  # noqa: E402
from transformers.models.olmoe.modeling_olmoe import load_balancing_loss_func  # noqa: E402


def _pair(seed=0):
    cfg = get_config("debug-olmoe")
    torch.manual_seed(seed)
    ours = build_llama(cfg, dtype=torch.float32)
    hf = OlmoeForCausalLM(OlmoeConfig(**to_hf_config_dict(cfg))).float()
    hf.load_state_dict(ours.state_dict(), strict=True)
    return cfg, ours, hf


def _hf_loss(hf, ids, coef):
    """HF's cross entropy, plus ``coef`` times ``load_balancing_loss_func`` of the raw router logits (x @ W_g^T at
    every layer's gate), which applies the softmax itself."""
    gate_in = []
    hooks = [layer.mlp.gate.register_forward_hook(lambda m, args, out: gate_in.append((m, args[0])))
             for layer in hf.model.layers]
    try:
        out = hf(ids, labels=ids)
    finally:
        for h in hooks:
            h.remove()
    logits = tuple(x.reshape(-1, x.shape[-1]) @ m.weight.t() for m, x in gate_in)
    aux = load_balancing_loss_func(logits, hf.config.num_experts, hf.config.num_experts_per_tok)
    return out, out.loss + coef * aux, aux


@pytest.mark.parametrize("coef", [0.0, 0.01])
def test_matches_transformers_logits_loss_and_grads(coef):
    cfg, ours, hf = _pair()
    ours.router_aux_loss_coef = coef
    ids = torch.randint(0, cfg.vocab_size, (2, 96), generator=torch.Generator().manual_seed(1))
    out = ours(ids, labels=ids, return_logits=True)
    out.loss.backward()
    hf_out, hf_loss, hf_aux = _hf_loss(hf, ids, coef)
    hf_loss.backward()
    torch.testing.assert_close(out.logits, hf_out.logits, rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(out.loss, hf_loss, rtol=1e-6, atol=1e-6)
    if coef:
        torch.testing.assert_close(out.aux_loss, hf_aux, rtol=1e-6, atol=1e-6)
    hf_params = dict(hf.named_parameters())
    for n, p in ours.named_parameters():
        torch.testing.assert_close(p.grad, hf_params[n].grad, rtol=1e-4, atol=1e-6, msg=n)


def test_aux_loss_formula_matches_transformers():
    g = torch.Generator().manual_seed(3)
    E, k, T = 8, 2, 40
    logits = tuple(torch.randn(T, E, generator=g) for _ in range(3))
    counts, psums = [], []
    for lg in logits:
        p = torch.softmax(lg, -1)
        counts.append(torch.bincount(torch.topk(p, k, -1).indices.reshape(-1), minlength=E))
        psums.append(p.sum(0))
    torch.testing.assert_close(ref.router_aux_loss(counts, psums, T, E), load_balancing_loss_func(logits, E, k))


@pytest.mark.parametrize("name", ["allenai/OLMoE-1B-7B-0924", "debug-olmoe"])
def test_parameter_counts_equal_transformers(name):
    cfg = get_config(name)
    with torch.device("meta"):
        hf = OlmoeForCausalLM(OlmoeConfig(**to_hf_config_dict(cfg)))
    assert cfg.num_parameters() == sum(p.numel() for p in hf.parameters())
    if name.startswith("allenai"):
        assert cfg.num_parameters() == 6_919_161_856


def test_flat_order():
    order, fused = decoder_layout(get_config("debug-olmoe"))
    assert order == ("self_attn.q_proj.weight", "self_attn.k_proj.weight", "self_attn.v_proj.weight",
                     "self_attn.o_proj.weight", "mlp.gate.weight", "mlp.experts.gate_up_proj",
                     "mlp.experts.down_proj", "input_layernorm.weight", "post_attention_layernorm.weight",
                     "self_attn.q_norm.weight", "self_attn.k_norm.weight")
    assert fused == {"qkv": order[:3]}


def _olmoe_dict(**kw):
    d = OlmoeConfig(vocab_size=1024, hidden_size=256, intermediate_size=128, num_hidden_layers=2,
                    num_attention_heads=2, num_key_value_heads=2, num_experts=8, num_experts_per_tok=2).to_dict()
    d.update(kw)
    return d


def test_reads_hf_config():
    cfg = _from_hf_dict(_olmoe_dict(), "x")
    want = dataclasses.replace(get_config("debug-olmoe"), name="x", max_position_embeddings=4096)
    assert cfg == want
    assert cfg.full_qk_norm and cfg.moe and not cfg.post_norm
    assert _from_hf_dict(to_hf_config_dict(get_config("allenai/OLMoE-1B-7B-0924")), "y") == dataclasses.replace(
        get_config("allenai/OLMoE-1B-7B-0924"), name="y")


@pytest.mark.parametrize("key,value", [
    ("clip_qkv", 8.0), ("norm_topk_prob", True), ("attention_bias", True),
    ("rope_parameters", {"rope_type": "linear", "factor": 2.0, "rope_theta": 1e4}), ("attention_dropout", 0.1),
])
def test_refuses_unsupported_settings_by_key(key, value):
    with pytest.raises(ValueError, match=key):
        _from_hf_dict(_olmoe_dict(**{key: value}), "x")


def test_mixtral_stays_refused():
    with pytest.raises(ValueError, match="mixtral"):
        _from_hf_dict({"model_type": "mixtral"}, "x")


def test_tensor_parallel_and_fp8_refuse_moe():
    from distributed_training_guide_b200.parallel import strategies

    cfg = get_config("debug-olmoe")
    tp = strategies.TwoDParallel.__new__(strategies.TwoDParallel)
    tp.env, tp.mesh = None, None
    with pytest.raises(ValueError, match="mixture-of-experts"):
        tp.build_model(SimpleNamespace(), cfg)
    model = build_llama(cfg, dtype=torch.float32)
    with pytest.raises(ValueError, match="mixture-of-experts"):
        strategies._apply_fp8(SimpleNamespace(fp8=True), model)


def test_aux_loss_refuses_activation_checkpointing():
    cfg, ours, _ = _pair()
    ours.router_aux_loss_coef = 0.01
    ours.activation_checkpointing = True
    ids = torch.randint(0, cfg.vocab_size, (1, 32))
    with pytest.raises(ValueError, match="checkpointing"):
        ours(ids, labels=ids)


def test_activation_checkpointing_matches_plain():
    cfg, ours, _ = _pair()
    ids = torch.randint(0, cfg.vocab_size, (2, 64), generator=torch.Generator().manual_seed(5))
    ours(ids, labels=ids).loss.backward()
    plain = {n: p.grad.clone() for n, p in ours.named_parameters()}
    ours.zero_grad()
    ours.activation_checkpointing = True
    ours(ids, labels=ids).loss.backward()
    for n, p in ours.named_parameters():
        torch.testing.assert_close(p.grad, plain[n], rtol=1e-6, atol=1e-7, msg=n)


# ---------------------------------------------------------------------------------------------------------------
# checkpoints: the published per-expert layout in and out
# ---------------------------------------------------------------------------------------------------------------
def _save_per_expert(sd, cfg, path):
    import json
    import os

    from safetensors.torch import save_file

    from distributed_training_guide_b200.models import olmoe_layout

    os.makedirs(path, exist_ok=True)
    hf_sd = olmoe_layout.to_hf_state_dict(sd)
    assert "model.layers.0.mlp.experts.7.up_proj.weight" in hf_sd and not any("gate_up_proj" in k for k in hf_sd)
    save_file({k: v.contiguous() for k, v in hf_sd.items()}, os.path.join(path, "model.safetensors"))
    with open(os.path.join(path, "config.json"), "w") as fp:
        json.dump(to_hf_config_dict(cfg), fp)


def test_pretrained_reads_the_per_expert_layout(tmp_path):
    pytest.importorskip("safetensors")
    from distributed_training_guide_b200.tools.load_hf import maybe_load_pretrained

    cfg, ours, hf = _pair(seed=3)
    _save_per_expert(ours.state_dict(), cfg, str(tmp_path / "m"))
    torch.manual_seed(99)
    fresh = build_llama(get_config(str(tmp_path / "m")), dtype=torch.float32)
    assert maybe_load_pretrained(SimpleNamespace(model_name=str(tmp_path / "m"), pretrained="require"), model=fresh)
    for k, v in fresh.state_dict().items():
        assert torch.equal(v, ours.state_dict()[k]), k
    ids = torch.randint(0, cfg.vocab_size, (1, 64), generator=torch.Generator().manual_seed(2))
    with torch.no_grad():
        torch.testing.assert_close(fresh(ids, return_logits=True).logits, hf(ids).logits, rtol=1e-5, atol=1e-5)


def test_chapter04_checkpoint_consolidates_and_loads_with_from_pretrained(tmp_path):
    import subprocess
    import sys
    from pathlib import Path

    pytest.importorskip("safetensors")
    root = Path(__file__).resolve().parent.parent
    script = root / "04-fully-sharded-data-parallel" / "train_llm.py"
    cmd = [sys.executable, "-m", "torch.distributed.run", "--standalone", "--local-addr", "127.0.0.1",
           "--nproc-per-node", "2", str(script), "-d", "synthetic", "-m", "debug-olmoe", "-s", "128", "-b", "1",
           "--num-samples", "16", "--log-freq", "1", "--device", "cpu", "--save-dir", str(tmp_path), "-e", "exp",
           "--ckpt-freq", "2", "--lr", "1e-3", "--max-steps", "2"]
    r = subprocess.run(cmd, capture_output=True, text=True, cwd=str(script.parent), timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    from distributed_training_guide_b200.tools.consolidate import consolidate

    cfg = get_config("debug-olmoe")
    sd = torch.load(consolidate(str(tmp_path / "exp"), "debug-olmoe", world=2), weights_only=True)
    assert "model.layers.1.mlp.experts.3.gate_proj.weight" in sd and not any("gate_up_proj" in k for k in sd)
    out = tmp_path / "hf"
    out.mkdir()
    from safetensors.torch import save_file
    import json

    save_file({k: v.float().contiguous() for k, v in sd.items()}, str(out / "model.safetensors"))
    (out / "config.json").write_text(json.dumps(to_hf_config_dict(cfg)))
    hf, info = OlmoeForCausalLM.from_pretrained(str(out), output_loading_info=True, dtype=torch.float32)
    assert not info["missing_keys"] and not info["unexpected_keys"] and not info["mismatched_keys"], info
    ours = build_llama(cfg, dtype=torch.float32, init=False)
    from distributed_training_guide_b200.models import olmoe_layout

    ours.load_state_dict(olmoe_layout.from_hf_state_dict({k: v.float() for k, v in sd.items()},
                                                         ours.state_dict().keys(), cfg.num_experts), strict=True)
    ids = torch.randint(0, cfg.vocab_size, (1, 64), generator=torch.Generator().manual_seed(2))
    with torch.no_grad():
        torch.testing.assert_close(ours(ids, return_logits=True).logits, hf(ids).logits, rtol=1e-5, atol=1e-5)


# ---------------------------------------------------------------------------------------------------------------
# engines over gloo against one process, activation checkpointing off and on
# ---------------------------------------------------------------------------------------------------------------
S_DIST, LR_DIST, B_GLOBAL = 128, 5e-3, 4


def _batch(vocab, step, rank):
    g = torch.Generator().manual_seed(1000 * step + rank)
    ids = torch.randint(0, vocab, (1, S_DIST), generator=g)
    return {"input_ids": ids, "labels": ids.clone()}


def _train(rank, world, parallelism, steps, ckpt):
    from distributed_training_guide_b200.engine import TrainEngine

    torch.manual_seed(0)
    per = B_GLOBAL // world
    eng = TrainEngine.create("debug-olmoe", parallelism=parallelism, batch_size=per, seq_length=S_DIST, device="cpu",
                             lr=LR_DIST, checkpoint_activations=ckpt)
    dp_rank = eng.strategy.dp_rank if world > 1 else 0
    losses = []
    for i in range(steps):
        parts = [_batch(eng.config.vocab_size, 0, dp_rank * per + j) for j in range(per)]   # one batch: the loss falls
        losses.append(float(eng.step({k: torch.cat([p[k] for p in parts]) for k in parts[0]})))
    return losses


@pytest.mark.parametrize("ckpt", [False, True])
@pytest.mark.parametrize("parallelism", ["ddp", "fsdp"])
def test_distributed_olmoe_matches_single_process(parallelism, ckpt):
    import numpy as np
    from dist_utils import run_distributed

    steps = 3
    res = run_distributed(_train, world=2, args=(parallelism, steps, ckpt), timeout=600)
    want = _train(0, 1, "single", steps, ckpt)
    for i in range(steps):
        mean = float(np.mean([r[i] for r in res]))
        assert abs(mean - want[i]) < 2e-2, (parallelism, ckpt, i, [r[i] for r in res], want[i])
    assert want[-1] < want[0], want   # the steps train: the comparison is not of three untouched models


def test_router_aux_loss_flag():
    from distributed_training_guide_b200.parallel.strategies import _apply_router_aux_loss
    from distributed_training_guide_b200.utils.cli import get_parser

    a = get_parser("01-single-gpu").parse_args(["-d", "synthetic", "-m", "debug-olmoe", "--router-aux-loss-coef",
                                                "0.01"])
    model = build_llama(get_config("debug-olmoe"), dtype=torch.float32)
    _apply_router_aux_loss(a, model)
    assert model.router_aux_loss_coef == 0.01
    with pytest.raises(ValueError, match="mixture-of-experts"):
        _apply_router_aux_loss(a, build_llama(get_config("debug-llama"), dtype=torch.float32, device="meta",
                                              init=False))


@pytest.mark.parametrize("coef", [0.0, 0.01])
def test_model_under_an_engine_is_freed(coef):
    """A layer must not keep its router statistics past the forward: their autograd graph reaches the engine's
    boundaries, whose callbacks hold the engine and so the model, and a reference from the layer would close a cycle
    through autograd nodes that the garbage collector cannot see (the model, and with FSDP the symmetric gradient
    slots its parameters point into, would never be freed)."""
    import gc
    import weakref

    from distributed_training_guide_b200.parallel.ddp import boundary

    class Hooks:   # the engines' hook protocol, with a boundary in front of every layer bound to the engine
        def pre_forward(self, model):
            pass

        def pre_layer(self, i, layer, x, residual):
            return boundary(lambda: self.model, x, residual)

        def post_layer(self, i, layer, x, residual):
            return x, residual

        def pre_head(self, x, residual):
            return x, residual

    cfg = get_config("debug-olmoe")
    model = build_llama(cfg, dtype=torch.float32)
    model.router_aux_loss_coef = coef
    model.engine = Hooks()
    model.engine.model = model
    ids = torch.randint(0, cfg.vocab_size, (1, 32), generator=torch.Generator().manual_seed(0))
    model(input_ids=ids, labels=ids).loss.backward()
    assert all(layer.router_stats is None for layer in model.model.layers)
    alive = weakref.ref(model.model.layers[0].mlp.gate.weight)
    del model
    gc.collect()
    assert alive() is None, "the model outlived its last reference"
