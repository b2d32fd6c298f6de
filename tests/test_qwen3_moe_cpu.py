"""Qwen3-MoE on the CPU: the fp32 reference path against transformers' ``Qwen3MoeForCausalLM`` (logits, loss and every
parameter's gradient, with ``norm_topk_prob`` true and false and the load-balancing loss off and on), the registry's
parameter counts, reading and refusing HF configs, the flat-buffer layout, checkpoints in the per-expert layout,
two-rank DDP and FSDP, and ``ref.moe(norm_topk_prob=True)`` against an independent fp64 computation."""
import dataclasses
import math
from types import SimpleNamespace

import pytest
import torch

from distributed_training_guide_b200.models.configs import _from_hf_dict, get_config, to_hf_config_dict
from distributed_training_guide_b200.models.llama import build_llama, decoder_layout
from distributed_training_guide_b200.ops import reference as ref
from test_gpu_moe_reference import PATH_SLACK, U
from test_gpu_qwen3_moe_reference import NORM_MUTATIONS, _norm_path_bound, moe_fixed_grads_norm

transformers = pytest.importorskip("transformers")
from transformers import Qwen3MoeConfig, Qwen3MoeForCausalLM  # noqa: E402
from transformers.models.qwen3_moe.modeling_qwen3_moe import load_balancing_loss_func  # noqa: E402

NAMES = ("y", "psum", "dx", "d_gate", "d_gate_up", "d_down")


def _pair(seed=0, norm=True):
    cfg = dataclasses.replace(get_config("debug-qwen3-moe"), norm_topk_prob=norm)
    torch.manual_seed(seed)
    ours = build_llama(cfg, dtype=torch.float32)
    hf = Qwen3MoeForCausalLM(Qwen3MoeConfig(**to_hf_config_dict(cfg))).float()
    hf.load_state_dict(ours.state_dict(), strict=True)
    assert hf.config.norm_topk_prob == norm and hf.config.head_dim == 128
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
@pytest.mark.parametrize("norm", [True, False])
def test_matches_transformers_logits_loss_and_grads(norm, coef):
    cfg, ours, hf = _pair(norm=norm)
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


def test_renormalisation_changes_the_model():
    """The flag is not a no-op: the same weights give other logits with and without it."""
    _, a, _ = _pair(norm=True)
    cfg, b, _ = _pair(norm=False)
    ids = torch.randint(0, cfg.vocab_size, (1, 32), generator=torch.Generator().manual_seed(4))
    with torch.no_grad():
        assert not torch.allclose(a(ids, return_logits=True).logits, b(ids, return_logits=True).logits, atol=1e-4)


@pytest.mark.parametrize("name,total", [("Qwen/Qwen3-30B-A3B", 30_532_122_624),
                                        ("Qwen/Qwen3-30B-A3B-Base", 30_532_122_624),
                                        ("Qwen/Qwen3-235B-A22B", 235_093_634_560), ("debug-qwen3-moe", None)])
def test_parameter_counts_equal_transformers(name, total):
    cfg = get_config(name)
    with torch.device("meta"):
        hf = Qwen3MoeForCausalLM(Qwen3MoeConfig(**to_hf_config_dict(cfg)))
    assert cfg.num_parameters() == sum(p.numel() for p in hf.parameters())
    if total is not None:
        assert cfg.num_parameters() == total


@pytest.mark.parametrize("name", ["Qwen/Qwen3-30B-A3B", "Qwen/Qwen3-235B-A22B", "debug-qwen3-moe"])
def test_registry_entries(name):
    cfg = get_config(name)
    assert cfg.arch == "qwen3_moe" and cfg.moe and cfg.qk_norm and not cfg.full_qk_norm and cfg.norm_topk_prob
    assert cfg.head_dim == 128 and not cfg.tie_word_embeddings and cfg.rms_norm_eps == 1e-6 and cfg.rope_theta == 1e6
    if name != "debug-qwen3-moe":
        assert cfg.max_position_embeddings == 40960
        assert (cfg.num_experts, cfg.num_experts_per_tok, cfg.vocab_size) == (128, 8, 151936)


def test_olmoe_configs_keep_raw_routing():
    cfg = get_config("allenai/OLMoE-1B-7B-0924")
    assert not cfg.norm_topk_prob and to_hf_config_dict(cfg)["norm_topk_prob"] is False


def test_flat_order():
    order, fused = decoder_layout(get_config("debug-qwen3-moe"))
    assert order == ("self_attn.q_proj.weight", "self_attn.k_proj.weight", "self_attn.v_proj.weight",
                     "self_attn.o_proj.weight", "mlp.gate.weight", "mlp.experts.gate_up_proj",
                     "mlp.experts.down_proj", "input_layernorm.weight", "post_attention_layernorm.weight",
                     "self_attn.q_norm.weight", "self_attn.k_norm.weight")
    assert fused == {"qkv": order[:3]}
    m = build_llama(get_config("debug-qwen3-moe"), dtype=torch.float32, device="meta", init=False)
    layer = m.model.layers[0]
    assert layer.self_attn.q_norm.weight.shape == (128,) and layer.mlp.experts.gate_up_proj.shape == (16, 256, 256)
    assert layer.mlp.experts.down_proj.shape == (16, 256, 128) and layer.mlp.norm_topk_prob


def _qwen3_moe_dict(**kw):
    d = Qwen3MoeConfig(vocab_size=1024, hidden_size=256, moe_intermediate_size=128, num_hidden_layers=2,
                       num_attention_heads=4, num_key_value_heads=2, head_dim=128, num_experts=16,
                       num_experts_per_tok=4, norm_topk_prob=True, max_position_embeddings=2048,
                       rope_parameters={"rope_type": "default", "rope_theta": 1e6}).to_dict()
    d.update(kw)
    return d


def test_reads_hf_config():
    cfg = _from_hf_dict(_qwen3_moe_dict(), "x")
    assert cfg == dataclasses.replace(get_config("debug-qwen3-moe"), name="x")
    assert not _from_hf_dict(_qwen3_moe_dict(norm_topk_prob=False), "x").norm_topk_prob
    d = _qwen3_moe_dict()
    del d["norm_topk_prob"]                                        # Qwen3MoeConfig's default: raw weights
    assert not _from_hf_dict(d, "x").norm_topk_prob
    for name in ("Qwen/Qwen3-30B-A3B", "Qwen/Qwen3-235B-A22B"):
        assert _from_hf_dict(to_hf_config_dict(get_config(name)), "y") == dataclasses.replace(get_config(name), name="y")
    # training options, not part of the model
    assert _from_hf_dict(_qwen3_moe_dict(router_aux_loss_coef=0.5, output_router_logits=True), "x") == cfg


@pytest.mark.parametrize("key,value", [
    ("mlp_only_layers", [1]), ("decoder_sparse_step", 2), ("use_sliding_window", True),
    ("layer_types", ["full_attention", "sliding_attention"]), ("attention_bias", True),
    ("rope_parameters", {"rope_type": "yarn", "factor": 4.0, "rope_theta": 1e6}), ("attention_dropout", 0.1),
    ("hidden_act", "gelu"), ("num_experts", 512), ("head_dim", 64),
])
def test_refuses_unsupported_settings_by_key(key, value):
    with pytest.raises(ValueError, match=key):
        _from_hf_dict(_qwen3_moe_dict(**{key: value}), "x")


def test_tensor_parallel_and_fp8_refuse_qwen3_moe():
    from distributed_training_guide_b200.parallel import strategies

    cfg = get_config("debug-qwen3-moe")
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
# the reference MoE with renormalised weights against fp64
# ---------------------------------------------------------------------------------------------------------------
def _inputs(T=160, E=16, k=4, H=64, I=32, seed=0):
    g = torch.Generator().manual_seed(seed)
    f64 = torch.float64
    x = torch.randn(T, H, generator=g, dtype=f64)
    gate_w = torch.randn(E, H, generator=g, dtype=f64) / math.sqrt(H)
    gate_up = torch.randn(E, 2 * I, H, generator=g, dtype=f64) / math.sqrt(H)
    down = torch.randn(E, H, I, generator=g, dtype=f64) / math.sqrt(I)
    top = torch.softmax(x @ gate_w.t(), -1).topk(k + 1, dim=-1).values
    x = x[(top[:, k - 1] - top[:, k]) > 1e-3]                      # fp32 and fp64 choose the same experts
    dy = torch.randn(x.shape[0], H, generator=g, dtype=f64)
    dpsum = torch.randn(E, generator=g, dtype=f64) * math.sqrt(H)
    idx = torch.softmax(x @ gate_w.t(), -1).topk(k, dim=-1).indices
    return x, gate_w, gate_up, down, k, dy, dpsum, idx


def _independent_fp64(x, gate_w, gate_up, down, k):
    """y of the renormalised MoE token by token in fp64, written without the reference's helpers."""
    y = torch.zeros_like(x)
    for t in range(x.shape[0]):
        p = torch.softmax(gate_w @ x[t], -1)
        order = sorted(range(p.numel()), key=lambda e: -float(p[e]))[:k]
        s = sum(float(p[e]) for e in order)
        for e in order:
            gu = gate_up[e] @ x[t]
            g, u = gu[:gu.numel() // 2], gu[gu.numel() // 2:]
            y[t] += (float(p[e]) / s) * (down[e] @ (g * torch.sigmoid(g) * u))
    return y


def test_reference_norm_matches_independent_fp64():
    x, gate_w, gate_up, down, k, dy, dpsum, idx = _inputs()
    assert x.shape[0] > 100
    y, p = ref.moe(x.float(), gate_w.float(), gate_up.float(), down.float(), k, norm_topk_prob=True)
    want = _independent_fp64(x, gate_w, gate_up, down, k)
    torch.testing.assert_close(y.double(), want, rtol=1e-4, atol=1e-5 * want.abs().max().item())
    raw, _ = ref.moe(x.float(), gate_w.float(), gate_up.float(), down.float(), k)
    assert not torch.allclose(raw.double(), want, atol=1e-3)       # the flag reaches the computation


def test_fixed_routing_norm_reference_equals_ops_reference():
    """The fp64 graph the GPU test holds ops.moe(norm_topk_prob=True) to equals ref.moe in y, psum and every
    gradient."""
    x, gate_w, gate_up, down, k, dy, dpsum, idx = _inputs(seed=1)
    got = dict(zip(NAMES, moe_fixed_grads_norm(x, gate_w, gate_up, down, idx, dy, dpsum)))
    leaves = [t.float().requires_grad_() for t in (x, gate_w, gate_up, down)]
    y, p = ref.moe(*leaves, k, norm_topk_prob=True)
    grads = torch.autograd.grad((y, p.sum(0)), leaves, (dy.float(), dpsum.float()))
    want = dict(zip(NAMES, (y.detach(), p.sum(0).detach()) + grads))
    for n in NAMES:
        scale = want[n].abs().max().item()
        torch.testing.assert_close(got[n], want[n].double(), rtol=1e-4, atol=1e-5 * scale, msg=n)


def test_norm_bound_pass_values_equal_autograd_and_reject_mistakes():
    """With dy = y (the gradient of |y|^2 / 2) the routing weights' gradients share a sign, so dropping the
    ``- sum w dw`` term moves dx by more than two bounds; a random dy lets that sum cancel."""
    x, gate_w, gate_up, down, k, dy, dpsum, idx = _inputs(seed=2)
    dy = moe_fixed_grads_norm(x, gate_w, gate_up, down, idx, dy, dpsum)[0]
    auto = dict(zip(NAMES, moe_fixed_grads_norm(x, gate_w, gate_up, down, idx, dy, dpsum)))
    p = torch.softmax(x @ gate_w.t(), -1)
    bounds = _norm_path_bound(x, gate_w, gate_up, down, idx, p, dy, dpsum, torch.float64)
    for n, (value, bound) in bounds.items():
        torch.testing.assert_close(value, auto[n], rtol=1e-10, atol=1e-12, msg=n)
        assert bool((bound >= value.abs()).all()), n
    for m in NORM_MUTATIONS:
        bad = dict(zip(NAMES, moe_fixed_grads_norm(x, gate_w, gate_up, down, idx, dy, dpsum, mutate=m)))
        caught = [n for n, (_, b) in bounds.items() if ((bad[n] - auto[n]).abs() > 2 * U * PATH_SLACK * b).any()]
        assert caught, m


# ---------------------------------------------------------------------------------------------------------------
# checkpoints: the published per-expert layout in and out
# ---------------------------------------------------------------------------------------------------------------
def test_pretrained_reads_the_per_expert_layout(tmp_path):
    pytest.importorskip("safetensors")
    import json
    import os

    from safetensors.torch import save_file

    from distributed_training_guide_b200.models import olmoe_layout
    from distributed_training_guide_b200.tools.load_hf import maybe_load_pretrained

    cfg, ours, hf = _pair(seed=3)
    path = str(tmp_path / "m")
    os.makedirs(path)
    hf_sd = olmoe_layout.to_hf_state_dict(ours.state_dict())
    assert "model.layers.0.mlp.experts.15.up_proj.weight" in hf_sd and not any("gate_up_proj" in k for k in hf_sd)
    save_file({k: v.contiguous() for k, v in hf_sd.items()}, os.path.join(path, "model.safetensors"))
    with open(os.path.join(path, "config.json"), "w") as fp:
        json.dump(to_hf_config_dict(cfg), fp)
    torch.manual_seed(99)
    loaded_cfg = get_config(path)
    assert loaded_cfg.arch == "qwen3_moe" and loaded_cfg.norm_topk_prob
    fresh = build_llama(loaded_cfg, dtype=torch.float32)
    assert maybe_load_pretrained(SimpleNamespace(model_name=path, pretrained="require"), model=fresh)
    for k, v in fresh.state_dict().items():
        assert torch.equal(v, ours.state_dict()[k]), k
    ids = torch.randint(0, cfg.vocab_size, (1, 64), generator=torch.Generator().manual_seed(2))
    with torch.no_grad():
        torch.testing.assert_close(fresh(ids, return_logits=True).logits, hf(ids).logits, rtol=1e-5, atol=1e-5)


def test_chapter04_checkpoint_consolidates_and_loads_with_from_pretrained(tmp_path):
    import json
    import subprocess
    import sys
    from pathlib import Path

    pytest.importorskip("safetensors")
    from safetensors.torch import save_file

    from distributed_training_guide_b200.models import olmoe_layout
    from distributed_training_guide_b200.tools.consolidate import consolidate

    root = Path(__file__).resolve().parent.parent
    script = root / "04-fully-sharded-data-parallel" / "train_llm.py"
    cmd = [sys.executable, "-m", "torch.distributed.run", "--standalone", "--local-addr", "127.0.0.1",
           "--nproc-per-node", "2", str(script), "-d", "synthetic", "-m", "debug-qwen3-moe", "-s", "128", "-b", "1",
           "--num-samples", "16", "--log-freq", "1", "--device", "cpu", "--save-dir", str(tmp_path), "-e", "exp",
           "--ckpt-freq", "2", "--lr", "1e-3", "--max-steps", "2"]
    r = subprocess.run(cmd, capture_output=True, text=True, cwd=str(script.parent), timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    cfg = get_config("debug-qwen3-moe")
    sd = torch.load(consolidate(str(tmp_path / "exp"), "debug-qwen3-moe", world=2), weights_only=True)
    assert "model.layers.1.mlp.experts.15.gate_proj.weight" in sd and not any("gate_up_proj" in k for k in sd)
    out = tmp_path / "hf"
    out.mkdir()
    save_file({k: v.float().contiguous() for k, v in sd.items()}, str(out / "model.safetensors"))
    (out / "config.json").write_text(json.dumps(to_hf_config_dict(cfg)))
    hf, info = Qwen3MoeForCausalLM.from_pretrained(str(out), output_loading_info=True, dtype=torch.float32)
    assert not info["missing_keys"] and not info["unexpected_keys"] and not info["mismatched_keys"], info
    assert hf.config.norm_topk_prob
    ours = build_llama(cfg, dtype=torch.float32, init=False)
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
    eng = TrainEngine.create("debug-qwen3-moe", parallelism=parallelism, batch_size=per, seq_length=S_DIST,
                             device="cpu", lr=LR_DIST, checkpoint_activations=ckpt)
    dp_rank = eng.strategy.dp_rank if world > 1 else 0
    losses = []
    for i in range(steps):
        parts = [_batch(eng.config.vocab_size, 0, dp_rank * per + j) for j in range(per)]
        losses.append(float(eng.step({k: torch.cat([p[k] for p in parts]) for k in parts[0]})))
    return losses


@pytest.mark.parametrize("ckpt", [False, True])
@pytest.mark.parametrize("parallelism", ["ddp", "fsdp"])
def test_distributed_qwen3_moe_matches_single_process(parallelism, ckpt):
    import numpy as np
    from dist_utils import run_distributed

    steps = 3
    res = run_distributed(_train, world=2, args=(parallelism, steps, ckpt), timeout=600)
    want = _train(0, 1, "single", steps, ckpt)
    for i in range(steps):
        mean = float(np.mean([r[i] for r in res]))
        assert abs(mean - want[i]) < 2e-2, (parallelism, ckpt, i, [r[i] for r in res], want[i])
    assert want[-1] < want[0], want


def test_router_aux_loss_and_document_masking_flags():
    from distributed_training_guide_b200.parallel.strategies import _apply_router_aux_loss
    from distributed_training_guide_b200.utils.cli import get_parser

    a = get_parser("01-single-gpu").parse_args(["-d", "synthetic", "-m", "debug-qwen3-moe", "--router-aux-loss-coef",
                                                "0.01", "--document-masking"])
    model = build_llama(get_config("debug-qwen3-moe"), dtype=torch.float32)
    _apply_router_aux_loss(a, model)
    assert model.router_aux_loss_coef == 0.01 and a.document_masking
