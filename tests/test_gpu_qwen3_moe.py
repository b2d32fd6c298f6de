"""Qwen3-MoE training on one GPU: single-GPU steps of debug-qwen3-moe (renormalised routing weights, per-head
QK-norm at head_dim 128) against an fp32 reference model parameter by parameter (plain, with packed documents and with
activation checkpointing), the load-balancing loss, and chapter 01.  The gradients are held to the bf16 run's distance
from fp32, as for OLMoE (``test_gpu_olmoe._check_moe_grads``)."""
import math

import pytest
import torch

from test_gpu_chapters import ROOT, _run
from test_gpu_olmoe import _check_moe_grads
from test_gpu_qwen3 import _plain_grads_docmask, _positions_from_starts
from test_gpu_step_reference import (LOSS_FACTOR, LOSS_SLACK, _capture_buckets, _engine, _engine_grads,
                                     _plain_model_grads, _print_report)

pytestmark = pytest.mark.gpu

CASE = dict(model="debug-qwen3-moe", B=2, S=256, overrides={})


@pytest.mark.parametrize("ckpt", [False, True])
def test_qwen3_moe_steps_match_fp32_reference(ckpt, monkeypatch):
    report = []
    with _engine(monkeypatch, CASE) as eng:
        assert eng.config.norm_topk_prob and eng.config.qk_norm
        eng.model.activation_checkpointing = ckpt
        rec = _capture_buckets(eng)
        for step in (1, 2):
            batch = eng.synthetic_batch(seed=step - 1)
            weights = {n: p.detach().clone() for n, p in eng.model.named_parameters()}
            loss = float(eng.step(batch))
            torch.cuda.synchronize()
            (l32,), g32 = _plain_model_grads(eng.config, {n: w.float() for n, w in weights.items()}, [batch],
                                             torch.float32, monkeypatch)
            (l16,), g16 = _plain_model_grads(eng.config, weights, [batch], torch.bfloat16, monkeypatch)
            assert abs(loss - l32) <= LOSS_FACTOR * abs(l16 - l32) + LOSS_SLACK, (step, loss, l32, l16)
            if step == 1:   # as for OLMoE: after an update, expert flips between bf16 and fp32 vary; step 2 by loss
                _check_moe_grads(f"s{step}", _engine_grads(eng, rec), g32, g16, report)
    _print_report(f"qwen3_moe ckpt={ckpt}", report)


def test_qwen3_moe_packed_step_matches_fp32_reference(monkeypatch):
    from distributed_training_guide_b200.engine import TrainEngine

    B, S = 2, 512
    eng = TrainEngine.create("debug-qwen3-moe", parallelism="single", batch_size=B, seq_length=S, lr=5e-3,
                             device="cuda", document_masking=True)
    try:
        weights = {n: p.detach().clone() for n, p in eng.model.named_parameters()}
        ids = torch.randint(0, eng.config.vocab_size, (B, S), generator=torch.Generator().manual_seed(7))
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
    _check_moe_grads("docmask", grads, g32, g16, report)
    _print_report("qwen3_moe packed step", report)


def test_qwen3_moe_aux_loss_gradient_matches_fp32_reference(monkeypatch):
    from distributed_training_guide_b200 import _ext
    from distributed_training_guide_b200.models.configs import get_config
    from distributed_training_guide_b200.models.llama import build_llama

    cfg = get_config("debug-qwen3-moe")
    torch.manual_seed(0)
    m16 = build_llama(cfg, dtype=torch.bfloat16, device="cuda")
    ids = torch.randint(0, cfg.vocab_size, (2, 256), device="cuda")
    grads, aux = {}, {}
    for kind in ("kernels", "fp32", "torch-bf16"):
        m = m16 if kind == "kernels" else build_llama(cfg, dtype=torch.float32 if kind == "fp32" else torch.bfloat16,
                                                      device="cuda", init=False)
        if m is not m16:
            m.load_state_dict({n: p.to(next(m.parameters()).dtype) for n, p in m16.state_dict().items()})
        m.router_aux_loss_coef = 0.01
        with monkeypatch.context() as mp:
            if kind == "torch-bf16":
                mp.setattr(_ext, "_forced", {"all"})
            n0 = _ext.launch_count()
            out = m(ids, labels=ids)
            out.loss.backward()
            if kind == "kernels":
                assert _ext.launch_count() > n0, "the bf16 model did not run the sm_90a kernels"
        aux[kind] = out.aux_loss.item()
        grads[kind] = {n: p.grad.float() for n, p in m.named_parameters()}
    assert abs(aux["kernels"] - aux["fp32"]) <= 2 * abs(aux["torch-bf16"] - aux["fp32"]) + 1e-3 * aux["fp32"], aux
    _check_moe_grads("aux", grads["kernels"], grads["fp32"], grads["torch-bf16"], [])


def test_chapter01_qwen3_moe_runs(tmp_path):
    args = ["-d", "synthetic", "-m", "debug-qwen3-moe", "-s", "256", "-b", "2", "--num-samples", "16", "--log-freq",
            "1", "-e", "exp", "--lr", "1e-3", "--save-dir", str(tmp_path), "--max-steps", "3",
            "--router-aux-loss-coef", "0.001"]
    recs, _ = _run(ROOT / "01-single-gpu" / "train_llm.py", args)
    losses = [r["running_loss"] for r in sorted(recs, key=lambda r: r["global_step"])]
    assert len(losses) == 3 and all(math.isfinite(x) and 0 < x < 20 for x in losses)
