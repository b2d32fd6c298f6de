"""Mistral / sliding-window attention on the CPU: the reference mask against a brute-force loop, ``debug-mistral``
against ``transformers.MistralForCausalLM`` with the same weights, the HF config round trip and a saved HF checkpoint
loaded through ``--pretrained``, the registry, and DDP / FSDP / TP over gloo against one process."""
import json

import numpy as np
import pytest
import torch

from dist_utils import run_distributed
from distributed_training_guide_b200 import ops
from distributed_training_guide_b200.models import build_model, get_config, to_hf_config_dict
from distributed_training_guide_b200.ops import reference as ref


# ---------------------------------------------------------------------------------------------------------------
# the mask
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("window", [None, 1, 2, 5, 13, 40, 41, 100])
@pytest.mark.parametrize("docs", [False, True])
def test_reference_mask_against_brute_force(window, docs):
    S = 41
    if docs:
        pos = torch.tensor([[i for i in range(7)] + [i for i in range(20)] + [i for i in range(14)],
                            [i for i in range(41)]])
    else:
        pos = torch.arange(S)[None].expand(2, S)
    ds = ops.document_starts(pos) if docs else None
    got = ref.document_mask(ds, S, window, device="cpu")
    B = 2 if docs else 1
    assert got.shape == (B, S, S) and got.dtype == torch.bool
    for b in range(B):
        for q in range(S):
            lo = int(ds[b, q]) if docs else 0
            if window is not None:
                lo = max(lo, q - window + 1)
            for k in range(S):
                assert bool(got[b, q, k]) == (lo <= k <= q), (b, q, k)


def test_reference_attention_window_equals_truncated_history():
    """Each query with a window W gives what plain causal attention gives on its W most recent tokens alone."""
    g = torch.Generator().manual_seed(0)
    S, W, nh, nkv = 30, 7, 4, 2
    q = torch.randn(1, S, nh, 16, generator=g, dtype=torch.float64)
    k = torch.randn(1, S, nkv, 16, generator=g, dtype=torch.float64)
    v = torch.randn(1, S, nkv, 16, generator=g, dtype=torch.float64)
    o = ref.attention(q, k, v, window=W)
    for t in range(S):
        a = max(0, t - W + 1)
        alone = ref.attention(q[:, a:t + 1], k[:, a:t + 1], v[:, a:t + 1])[:, -1]
        torch.testing.assert_close(o[:, t], alone, rtol=1e-5, atol=1e-6)


def test_attention_qkv_cpu_path_window():
    g = torch.Generator().manual_seed(1)
    qkv = torch.randn(2, 24, 6, 8, generator=g)
    o = ops.attention_qkv(qkv, 2, 2, window=5)
    torch.testing.assert_close(o, ref.attention(qkv[:, :, :2], qkv[:, :, 2:4], qkv[:, :, 4:], window=5))
    # a window of S or more is no window
    for w in (24, 25, 10 ** 6):
        assert torch.equal(ops.attention_qkv(qkv, 2, 2, window=w), ops.attention_qkv(qkv, 2, 2))
    # W = 1: every query sees only itself
    torch.testing.assert_close(ops.attention_qkv(qkv, 2, 2, window=1), qkv[:, :, 4:])
    # with document masking both bounds apply
    ds = ops.document_starts(torch.tensor([[0, 1, 2, 3, 4, 5, 6, 7, 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 0, 1, 2, 3, 4]]))
    ds = ds.expand(2, 24).contiguous()
    torch.testing.assert_close(ops.attention_qkv(qkv, 2, 2, doc_start=ds, window=5),
                               ref.attention(qkv[:, :, :2], qkv[:, :, 2:4], qkv[:, :, 4:], doc_start=ds, window=5))
    for bad in (0, -3, 2.5, True):
        with pytest.raises(ValueError, match="window"):
            ops.attention_qkv(qkv, 2, 2, window=bad)


# ---------------------------------------------------------------------------------------------------------------
# the model against transformers
# ---------------------------------------------------------------------------------------------------------------
def _hf_mistral(cfg, transformers, **over):
    d = {k: v for k, v in to_hf_config_dict(cfg).items() if k not in ("model_type", "architectures", "torch_dtype")}
    d.update(over)
    hf_cfg = transformers.MistralConfig(**d)
    hf_cfg._attn_implementation = "eager"
    return transformers.MistralForCausalLM(hf_cfg).float().eval()


def _peaked_debug_mistral():
    """fp32 ``debug-mistral`` whose q/k projections are scaled up so that attention is far from uniform: at the
    default init every query averages its keys almost evenly and a window would barely change the logits."""
    cfg = get_config("debug-mistral")
    torch.manual_seed(0)
    mine = build_model(cfg, dtype=torch.float32, device="cpu")
    with torch.no_grad():
        for layer in mine.model.layers:
            layer.self_attn.q_proj.weight.mul_(6.0)
            layer.self_attn.k_proj.weight.mul_(6.0)
    return cfg, mine


def test_debug_mistral_matches_transformers_fp32():
    transformers = pytest.importorskip("transformers")
    cfg, mine = _peaked_debug_mistral()
    assert cfg.arch == "mistral" and cfg.sliding_window == 192
    hf = _hf_mistral(cfg, transformers)
    missing, unexpected = hf.load_state_dict(mine.state_dict(), strict=False)
    assert not unexpected, unexpected
    assert all("rotary" in m or "inv_freq" in m for m in missing), missing   # names are HF's
    S = 320   # beyond the window of 192
    ids = torch.randint(0, cfg.vocab_size, (2, S), generator=torch.Generator().manual_seed(1))
    with torch.no_grad():
        out_mine = mine(input_ids=ids, labels=ids, return_logits=True)
        out_hf = hf(input_ids=ids, labels=ids)
        # the window matters at these weights: without it the late positions differ by far more than the tolerance
        no_win = _hf_mistral(cfg, transformers, sliding_window=None)
        no_win.load_state_dict(mine.state_dict(), strict=False)
        out_full = no_win(input_ids=ids)
    assert torch.allclose(out_mine.logits, out_hf.logits, atol=2e-4, rtol=1e-3), \
        (out_mine.logits - out_hf.logits).abs().max()
    assert abs(out_mine.loss.item() - out_hf.loss.item()) < 1e-4
    assert torch.allclose(out_hf.logits[:, :192], out_full.logits[:, :192], atol=2e-4, rtol=1e-3)
    assert (out_hf.logits[:, 192:] - out_full.logits[:, 192:]).abs().max() > 1e-2


# ---------------------------------------------------------------------------------------------------------------
# configs
# ---------------------------------------------------------------------------------------------------------------
def test_registry_mistral_7b():
    cfg = get_config("mistralai/Mistral-7B-v0.1")
    assert cfg.arch == "mistral" and cfg.sliding_window == 4096 and cfg.head_dim == 128
    assert (cfg.vocab_size, cfg.hidden_size, cfg.intermediate_size, cfg.num_hidden_layers) == (32000, 4096, 14336, 32)
    assert (cfg.num_attention_heads, cfg.num_key_value_heads, cfg.max_position_embeddings) == (32, 8, 32768)
    assert cfg.rope_theta == 1e4 and not cfg.tie_word_embeddings
    assert cfg.num_parameters() == 7_241_732_096
    model = build_model(get_config("debug-mistral"), dtype=torch.float32, device="meta")
    assert model.num_parameters() == get_config("debug-mistral").num_parameters()
    assert get_config("debug-mistral").sliding_window % 128 != 0


def _write_config(tmp_path, d):
    (tmp_path / "config.json").write_text(json.dumps(d))
    return str(tmp_path)


@pytest.mark.parametrize("name", ["mistralai/Mistral-7B-v0.1", "debug-mistral"])
def test_hf_config_round_trip(tmp_path, name):
    cfg = get_config(name)
    d = to_hf_config_dict(cfg)
    assert d["model_type"] == "mistral" and d["architectures"] == ["MistralForCausalLM"]
    assert d["sliding_window"] == cfg.sliding_window and d["head_dim"] == 128
    back = get_config(_write_config(tmp_path, d))
    assert back.to_dict() == {**cfg.to_dict(), "name": str(tmp_path)}
    transformers = pytest.importorskip("transformers")
    hf = transformers.MistralConfig(**{k: v for k, v in d.items() if k not in ("model_type", "architectures")})
    assert hf.sliding_window == cfg.sliding_window and hf.num_key_value_heads == cfg.num_key_value_heads


def test_hf_config_null_window_missing_window_and_head_dim(tmp_path):
    d = to_hf_config_dict(get_config("debug-mistral"))
    assert get_config(_write_config(tmp_path, {**d, "sliding_window": None})).sliding_window is None
    missing = {k: v for k, v in d.items() if k != "sliding_window"}
    assert get_config(_write_config(tmp_path, missing)).sliding_window == 4096   # MistralConfig's default
    assert get_config(_write_config(tmp_path, {k: v for k, v in d.items() if k != "head_dim"})).head_dim == 128
    with pytest.raises(ValueError, match="head_dim"):
        get_config(_write_config(tmp_path, {**d, "head_dim": 64}))
    with pytest.raises(ValueError, match="unsupported model_type"):
        get_config(_write_config(tmp_path, {**d, "model_type": "mixtral"}))


def test_llama_and_gpt2_payloads_unchanged():
    """The Llama and GPT-2 payloads keep exactly their keys: no window, no head_dim."""
    llama = to_hf_config_dict(get_config("debug-llama-gqa"))
    assert list(llama) == ["model_type", "architectures", "vocab_size", "hidden_size", "intermediate_size",
                           "num_hidden_layers", "num_attention_heads", "num_key_value_heads",
                           "max_position_embeddings", "rms_norm_eps", "rope_theta", "hidden_act",
                           "tie_word_embeddings", "attention_bias", "mlp_bias", "bos_token_id", "eos_token_id",
                           "torch_dtype"]
    assert get_config("meta-llama/Llama-2-7b-hf").sliding_window is None
    assert "sliding_window" not in to_hf_config_dict(get_config("gpt2"))


def test_pretrained_hf_mistral_checkpoint_loads(tmp_path):
    """A checkpoint written by ``transformers.MistralForCausalLM.save_pretrained`` (config.json + safetensors) loads
    through ``--pretrained`` unchanged: Mistral uses Llama's tensor names."""
    transformers = pytest.importorskip("transformers")
    pytest.importorskip("safetensors")
    from types import SimpleNamespace

    from distributed_training_guide_b200.tools.load_hf import maybe_load_pretrained

    cfg = get_config("debug-mistral")
    torch.manual_seed(5)
    hf = _hf_mistral(cfg, transformers)
    hf.save_pretrained(str(tmp_path / "m"), safe_serialization=True)
    loaded_cfg = get_config(str(tmp_path / "m"))
    assert loaded_cfg.arch == "mistral" and loaded_cfg.sliding_window == 192
    model = build_model(loaded_cfg, dtype=torch.float32, device="cpu")
    assert maybe_load_pretrained(SimpleNamespace(model_name=str(tmp_path / "m"), pretrained="require"), model=model)
    hf_sd = hf.state_dict()
    for k, v in model.state_dict().items():
        assert torch.equal(v, hf_sd[k]), k
    ids = torch.randint(0, cfg.vocab_size, (1, 256), generator=torch.Generator().manual_seed(2))
    with torch.no_grad():
        assert torch.allclose(model(input_ids=ids, return_logits=True).logits, hf(input_ids=ids).logits,
                              atol=2e-4, rtol=1e-3)


# ---------------------------------------------------------------------------------------------------------------
# DDP, FSDP and TP over gloo against one process
# ---------------------------------------------------------------------------------------------------------------
S_DIST = 256   # beyond debug-mistral's window of 192


def _batch(vocab, step, rank, B=1):
    g = torch.Generator().manual_seed(1000 * step + rank)
    ids = torch.randint(0, vocab, (B, S_DIST), generator=g)
    return {"input_ids": ids, "labels": ids.clone()}


def _record_windows():
    """Wrap ``ops.attention_qkv`` so that the windows the decoder layers pass are recorded."""
    seen = []
    orig = ops.attention_qkv

    def wrapped(*a, **kw):
        seen.append(kw.get("window"))
        return orig(*a, **kw)

    ops.attention_qkv = wrapped
    return seen


def _train_dist(rank, world, parallelism, steps):
    from distributed_training_guide_b200.engine import TrainEngine

    seen = _record_windows()
    torch.manual_seed(0)
    kw = {"tensor_parallel": world} if parallelism == "tp" else {}
    eng = TrainEngine.create("debug-mistral", parallelism=parallelism, batch_size=1, seq_length=S_DIST, device="cpu",
                             lr=1e-3, **kw)
    dp_rank = eng.strategy.dp_rank
    losses = [float(eng.step(_batch(eng.config.vocab_size, i, dp_rank))) for i in range(steps)]
    return losses, sorted(set(seen), key=str), eng.strategy.dp_size


def _single(steps, dp):
    from distributed_training_guide_b200.engine import TrainEngine

    torch.manual_seed(0)
    eng = TrainEngine.create("debug-mistral", parallelism="single", batch_size=dp, seq_length=S_DIST, device="cpu",
                             lr=1e-3)
    out = []
    for i in range(steps):
        parts = [_batch(eng.config.vocab_size, i, r) for r in range(dp)]
        out.append(float(eng.step({k: torch.cat([p[k] for p in parts]) for k in parts[0]})))
    return out


@pytest.mark.parametrize("parallelism", ["ddp", "fsdp", "tp"])
def test_distributed_mistral_matches_single_process(parallelism):
    steps, world = 3, 2
    res = run_distributed(_train_dist, world=world, args=(parallelism, steps), timeout=600)
    dp = res[0][2]
    ref_losses = _single(steps, dp)
    for losses, windows, _ in res:
        assert windows == [192], windows   # every decoder layer's attention got the window
    for i in range(steps):
        mean = float(np.mean([r[0][i] for r in res]))
        assert abs(mean - ref_losses[i]) < 2e-2, (parallelism, i, [r[0][i] for r in res], ref_losses[i])
    if parallelism == "tp":   # tensor-parallel peers agree on the loss
        assert np.allclose(res[0][0], res[1][0], atol=1e-5)
