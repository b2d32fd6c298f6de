"""Model parity on CPU: our Llama (reference ops path) against transformers' LlamaForCausalLM with the
same weights, parameter naming, init determinism across placements, GPT-2 plumbing."""
import pytest
import torch

from distributed_training_guide_b200.models import build_model, get_config, to_hf_config_dict


def test_llama_matches_transformers_fp32():
    transformers = pytest.importorskip("transformers")
    cfg = get_config("debug-llama-gqa")
    torch.manual_seed(0)
    mine = build_model(cfg, dtype=torch.float32, device="cpu")
    hf_cfg = transformers.LlamaConfig(**{k: v for k, v in to_hf_config_dict(cfg).items()
                                         if k not in ("model_type", "architectures", "torch_dtype")})
    hf = transformers.LlamaForCausalLM(hf_cfg).float()
    sd = mine.state_dict()
    missing, unexpected = hf.load_state_dict(sd, strict=False)
    assert not unexpected, unexpected
    assert all("rotary" in m or "inv_freq" in m for m in missing), missing  # names are HF's
    ids = torch.randint(0, cfg.vocab_size, (2, 48))
    out_mine = mine(input_ids=ids, labels=ids, return_logits=True)
    out_hf = hf(input_ids=ids, labels=ids)
    assert torch.allclose(out_mine.logits, out_hf.logits, atol=2e-4, rtol=1e-3)
    assert abs(out_mine.loss.item() - out_hf.loss.item()) < 1e-4


def test_init_is_placement_independent():
    """Same seed -> same weights whether built whole or as tensor-parallel slices."""
    from distributed_training_guide_b200.models.llama import TP_SHARD_DIM

    cfg = get_config("debug-llama-tp", num_hidden_layers=1)
    torch.manual_seed(3)
    full = build_model(cfg, dtype=torch.float32, device="cpu")
    shards = []
    for r in range(2):
        m = build_model(cfg, dtype=torch.float32, device="cpu", tp_size=2, init=False)
        m.tp_rank = r
        m.init_weights(seed=3)
        shards.append(dict(m.named_parameters()))
    for name, p in full.named_parameters():
        dim = next((d for k, d in TP_SHARD_DIM.items() if f"{k}.weight" in name), None)
        if dim is None:
            assert torch.equal(p, shards[0][name]) and torch.equal(p, shards[1][name]), name
        else:
            assert torch.equal(p, torch.cat([shards[0][name], shards[1][name]], dim=dim)), name


def test_gpt2_forward_backward_and_param_count():
    cfg = get_config("openai-community/gpt2")
    assert abs(cfg.num_parameters() - 124_439_808) < 10, cfg.num_parameters()
    model = build_model("debug-gpt2", dtype=torch.float32, device="cpu")
    ids = torch.randint(0, 512, (2, 32))
    out = model(input_ids=ids, labels=ids)
    out.loss.backward()
    assert out.logits.shape == (2, 32, 512) and torch.isfinite(out.loss)
    assert model.lm_head.weight is model.transformer.wte.weight  # tied


def test_registry_parameter_counts():
    assert abs(get_config("meta-llama/Llama-2-7b-hf").num_parameters() / 1e9 - 6.738) < 0.01
    assert abs(get_config("meta-llama/Meta-Llama-3-8B").num_parameters() / 1e9 - 8.030) < 0.01
    assert abs(get_config("meta-llama/Meta-Llama-3-70B").num_parameters() / 1e9 - 70.554) < 0.01
    assert abs(get_config("meta-llama/Llama-3.1-405B").num_parameters() / 1e9 - 405.85) < 0.1


def test_cross_entropy_without_valid_targets_is_zero():
    """The CPU path agrees with the CUDA kernel when every target is ignored: loss 0, zero gradient, no NaN; with
    valid targets it is the usual mean."""
    from distributed_training_guide_b200 import ops

    torch.manual_seed(0)
    logits = torch.randn(4, 16, requires_grad=True)
    loss = ops.cross_entropy(logits, torch.full((4,), -100))
    loss.backward()
    assert loss.item() == 0.0 and int(torch.count_nonzero(logits.grad)) == 0
    tgt = torch.tensor([1, -100, 3, 15])
    want = torch.nn.functional.cross_entropy(logits, tgt, ignore_index=-100)
    assert torch.allclose(ops.cross_entropy(logits, tgt), want, rtol=1e-6, atol=0)
