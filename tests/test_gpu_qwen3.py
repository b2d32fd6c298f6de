"""Qwen3 training on the GPU: three single-GPU steps of ``debug-qwen3`` (heads x head_dim = 512 over a hidden size
of 256), untied and tied, against an fp32 reference model parameter by parameter, including the QK-norm gains; a
packed-document step; and the chapter scripts with ``-m debug-qwen3``.  The helpers are those of
``test_gpu_step_reference.py``."""
import math

import pytest
import torch

from distributed_training_guide_b200 import _ext
from distributed_training_guide_b200.models.llama import build_llama
from test_gpu_chapters import ROOT, _run
from test_gpu_step_reference import (LOSS_FACTOR, LOSS_SLACK, _capture_buckets, _check_grads, _check_order,
                                     _check_update, _engine, _engine_grads, _fp32_matmuls, _plain_model_grads,
                                     _pre_step_state, _print_report)

pytestmark = pytest.mark.gpu

CONFIGS = {
    "qwen3-b2-s256": dict(model="debug-qwen3", B=2, S=256, overrides={}),
    "qwen3-b2-s256-tied": dict(model="debug-qwen3", B=2, S=256, overrides=dict(tie_word_embeddings=True)),
}


@pytest.mark.parametrize("case", list(CONFIGS))
def test_qwen3_step_matches_fp32_reference(case, monkeypatch):
    cfg = CONFIGS[case]
    report, worst = [], 0.0
    with _engine(monkeypatch, cfg) as eng:
        config = eng.config
        assert config.qk_norm and config.num_attention_heads * config.head_dim != config.hidden_size
        rec = _capture_buckets(eng)
        for step in (1, 2, 3):
            batch = eng.synthetic_batch(seed=step - 1)
            weights = {n: p.detach().clone() for n, p in eng.model.named_parameters()}
            assert any("q_norm" in n for n in weights) and any("k_norm" in n for n in weights)
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
            worst = max(worst, _check_grads(f"s{step}", grads, ref_grads, bf16_grads, report))
            _check_update(eng, rec, pre, step, lr)
    _print_report(f"{case}: per-parameter gradient error (worst ratio {worst:.2f})", report)


def _positions_from_starts(starts):
    S = starts.shape[1]
    idx = torch.arange(S).expand_as(starts)
    first = torch.where(starts, idx, torch.zeros_like(idx)).cummax(dim=1).values
    return idx - first


def _plain_grads_docmask(config, weights, batch, dtype, monkeypatch):
    model = build_llama(config, dtype=dtype, device="cuda", init=False)
    model.document_masking = True
    with torch.no_grad():
        for n, p in model.named_parameters():
            p.copy_(weights[n])
    with monkeypatch.context() as mp, _fp32_matmuls():
        if dtype == torch.bfloat16:
            mp.setattr(_ext, "_forced", {"all"})
        out = model(**{k: v.cuda() for k, v in batch.items()})
        out.loss.backward()
    return out.loss.item(), {n: p.grad.float() for n, p in model.named_parameters()}


def test_qwen3_packed_step_matches_fp32_reference(monkeypatch):
    """Per-token RoPE tables from ``position_ids`` reach the QK-norm kernel; attention stays inside documents."""
    from distributed_training_guide_b200.engine import TrainEngine

    B, S = 2, 512
    eng = TrainEngine.create("debug-qwen3", parallelism="single", batch_size=B, seq_length=S, lr=5e-3, device="cuda",
                             document_masking=True)
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
    _check_grads("docmask", grads, g32, g16, report)
    _print_report("qwen3 packed step", report)


CHAPTER_ARGS = ["-d", "synthetic", "-m", "debug-qwen3", "-s", "256", "-b", "2", "--num-samples", "32", "--log-freq",
                "1", "-e", "exp", "--lr", "1e-3", "--max-steps", "4"]


def _losses(recs):
    return [r["running_loss"] for r in sorted(recs, key=lambda r: r["global_step"])]


def test_chapter01_qwen3_on_gpu(tmp_path):
    recs, _ = _run(ROOT / "01-single-gpu" / "train_llm.py", CHAPTER_ARGS + ["--save-dir", str(tmp_path)])
    assert len(recs) == 4 and all(r["tokens_per_s"] > 0 for r in recs)
    assert all(0 < l < 20 and math.isfinite(l) for l in _losses(recs))


@pytest.mark.multigpu
@pytest.mark.parametrize("chapter", ["02-distributed-data-parallel", "04-fully-sharded-data-parallel",
                                     "06-tensor-parallel"])
def test_distributed_chapters_qwen3_match_single_gpu(tmp_path, chapter):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    single, _ = _run(ROOT / "01-single-gpu" / "train_llm.py", CHAPTER_ARGS + ["--save-dir", str(tmp_path / "one")])
    recs, _ = _run(ROOT / chapter / "train_llm.py", CHAPTER_ARGS + ["--save-dir", str(tmp_path / "many")], nproc=2)
    a, b = _losses(single), _losses(recs)
    # random tokens from the same initial weights: the first losses agree closely, and training stays finite
    assert abs(a[0] - b[0]) < 5e-2, (a, b)
    assert all(math.isfinite(x) and x < a[0] + 0.5 for x in b), (a, b)
