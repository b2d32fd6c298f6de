"""GPT-NeoX training on one GPU against an fp32 reference model.

Three single-GPU steps of debug-gpt-neox (head_dim 128, rotary 32) and debug-gpt-neox-d64 (head_dim 64, rotary 16),
parameter by parameter against an fp32 (and a bf16) model of the reference ops (the helpers of
``test_gpu_step_reference.py``); a packed-document step; --fp8 and --max-grad-norm; chapters 01 (with checkpoint and
resume), 02 and 04 under torchrun on one GPU."""
import json
import math

import pytest
import torch

from test_gpu_chapters import ROOT, _run
from test_gpu_qwen2 import _split_k_bias
from test_gpu_qwen3 import _plain_grads_docmask, _positions_from_starts
from test_gpu_step_reference import (LOSS_FACTOR, LOSS_SLACK, _capture_buckets, _check_grads, _check_order,
                                     _check_update, _engine, _engine_grads, _plain_model_grads, _pre_step_state,
                                     _print_report)

pytestmark = pytest.mark.gpu

CONFIGS = {
    "gpt-neox-b2-s256": dict(model="debug-gpt-neox", B=2, S=256, overrides={}),
    "gpt-neox-d64-b1-s512-tied": dict(model="debug-gpt-neox-d64", B=1, S=512,
                                      overrides=dict(tie_word_embeddings=True)),
}


@pytest.mark.parametrize("case", list(CONFIGS))
def test_gpt_neox_step_matches_fp32_reference(case, monkeypatch):
    cfg = CONFIGS[case]
    report, worst = [], 0.0
    with _engine(monkeypatch, cfg) as eng:
        config = eng.config
        assert config.parallel_residual and config.rotary_dim < config.head_dim
        rec = _capture_buckets(eng)
        for step in (1, 2, 3):
            batch = eng.synthetic_batch(seed=step - 1)
            weights = {n: p.detach().clone() for n, p in eng.model.named_parameters()}
            pre = _pre_step_state(eng)
            lr = eng.optimizer.lr
            rec["order"].clear()
            loss = float(eng.step(batch))
            torch.cuda.synchronize()
            _check_order(eng, rec, f"step {step}")
            (loss_ref,), ref_grads = _plain_model_grads(config, {n: w.float() for n, w in weights.items()}, [batch],
                                                        torch.float32, monkeypatch)
            (loss_bf16,), bf16_grads = _plain_model_grads(config, weights, [batch], torch.bfloat16, monkeypatch)
            assert abs(loss - loss_ref) <= LOSS_FACTOR * abs(loss_bf16 - loss_ref) + LOSS_SLACK, \
                (step, loss, loss_ref, loss_bf16)
            grads = _engine_grads(eng, rec)
            assert set(grads) == set(ref_grads)
            ref_grads, bf16_grads = _split_k_bias(grads, ref_grads, bf16_grads)   # k bias: softmax-invariant
            worst = max(worst, _check_grads(f"s{step}", grads, ref_grads, bf16_grads, report))
            _check_update(eng, rec, pre, step, lr)
    _print_report(f"{case}: per-parameter gradient error (worst ratio {worst:.2f})", report)


def test_gpt_neox_packed_step_matches_fp32_reference(monkeypatch):
    """Per-token partial RoPE tables and document masking; attention stays inside documents."""
    from distributed_training_guide_b200.engine import TrainEngine

    B, S = 2, 512
    eng = TrainEngine.create("debug-gpt-neox", parallelism="single", batch_size=B, seq_length=S, lr=5e-3,
                             device="cuda", document_masking=True)
    try:
        weights = {n: p.detach().clone() for n, p in eng.model.named_parameters()}
        g = torch.Generator().manual_seed(7)
        ids = torch.randint(0, eng.config.vocab_size, (B, S), generator=g)
        starts = torch.zeros(B, S, dtype=torch.bool)
        starts[0, [0, 1, 100, 128, 129, 300]] = True
        starts[1, [0, 256, 257, 511]] = True
        batch = {"input_ids": ids, "labels": ids.clone(), "position_ids": _positions_from_starts(starts)}
        rec = _capture_buckets(eng)
        loss = float(eng.step(batch))
        grads = _engine_grads(eng, rec)
    finally:
        eng.close()
    l32, g32 = _plain_grads_docmask(eng.config, weights, batch, torch.float32, monkeypatch)
    l16, g16 = _plain_grads_docmask(eng.config, weights, batch, torch.bfloat16, monkeypatch)
    assert abs(loss - l32) <= LOSS_FACTOR * abs(l16 - l32) + LOSS_SLACK, (loss, l32, l16)
    report = []
    g32, g16 = _split_k_bias(grads, g32, g16)
    _check_grads("docmask", grads, g32, g16, report)
    _print_report("gpt-neox packed step", report)


@pytest.mark.parametrize("flags", [dict(fp8=True), dict(max_grad_norm=0.5)])
def test_gpt_neox_flags_train_on_gpu(flags):
    """--fp8 (q|k|v, c_fc and both parallel_out GEMMs in fp8) and --max-grad-norm: finite losses that fall on a
    repeated batch, and every bias and norm parameter moves."""
    from distributed_training_guide_b200.engine import TrainEngine

    eng = TrainEngine.create("debug-gpt-neox", parallelism="single", batch_size=2, seq_length=256, lr=3e-3,
                             device="cuda", **flags)
    try:
        before = {n: p.detach().clone() for n, p in eng.model.named_parameters() if p.dim() == 1}
        batch = eng.synthetic_batch(seed=0)
        losses = [float(eng.step(batch)) for _ in range(4)]
        torch.cuda.synchronize()
        after = {n: p.detach() for n, p in eng.model.named_parameters() if p.dim() == 1}
    finally:
        eng.close()
    assert all(math.isfinite(l) for l in losses) and losses[-1] < losses[0], losses
    assert all(not torch.equal(before[n], after[n]) for n in before), \
        [n for n in before if torch.equal(before[n], after[n])]


CHAPTER_ARGS = ["-d", "synthetic", "-m", "debug-gpt-neox", "-s", "256", "-b", "2", "--num-samples", "32",
                "--log-freq", "1", "-e", "exp", "--lr", "1e-3", "--ckpt-freq", "3"]


def _losses(recs):
    return [r["running_loss"] for r in sorted(recs, key=lambda r: r["global_step"])]


def test_chapter01_gpt_neox_on_gpu_with_resume(tmp_path):
    script = ROOT / "01-single-gpu" / "train_llm.py"
    args = CHAPTER_ARGS + ["--save-dir", str(tmp_path)]
    recs, _ = _run(script, args + ["--max-steps", "3"])
    assert len(recs) == 3 and all(r["tokens_per_s"] > 0 for r in recs)
    assert all(0 < l < 20 and math.isfinite(l) for l in _losses(recs))
    assert json.loads((tmp_path / "exp" / "state.json").read_text())["global_step"] == 3
    recs2, log = _run(script, args + ["--max-steps", "6"])
    assert "Resumed=True" in log and recs2[-1]["global_step"] == 6
    assert all(0 < l < 20 and math.isfinite(l) for l in _losses(recs2))


@pytest.mark.parametrize("chapter", ["02-distributed-data-parallel", "04-fully-sharded-data-parallel"])
def test_distributed_chapters_gpt_neox_on_one_gpu(tmp_path, chapter):
    args = CHAPTER_ARGS + ["--max-steps", "4"]
    single, _ = _run(ROOT / "01-single-gpu" / "train_llm.py", args + ["--save-dir", str(tmp_path / "one")])
    recs, _ = _run(ROOT / chapter / "train_llm.py", args + ["--save-dir", str(tmp_path / "many")], nproc=1)
    a, b = _losses(single), _losses(recs)
    assert abs(a[0] - b[0]) < 5e-2, (a, b)
    assert all(math.isfinite(x) and x < a[0] + 0.5 for x in b), (a, b)
