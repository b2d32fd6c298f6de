"""Qwen2 training on the GPU: three single-GPU steps of ``debug-qwen2`` (q/k/v biases; head_dim 64, and a head_dim 128
variant) untied and tied, against an fp32 reference model parameter by parameter, bias gradients included; a
packed-document step; an ``--fp8`` step; a ``--max-grad-norm`` step whose norm is checked against
``clip_grad_norm_`` on the fp32 model; and the chapter scripts with ``-m debug-qwen2``.  The helpers are those of
``test_gpu_step_reference.py``."""
import math

import pytest
import torch

from test_gpu_chapters import ROOT, _run
from test_gpu_qwen3 import _plain_grads_docmask, _positions_from_starts
from test_gpu_step_reference import (GRAD_CEILING, LOSS_FACTOR, LOSS_SLACK, _capture_buckets, _check_grads,
                                     _check_order, _check_update, _engine, _engine_grads, _plain_model_grads,
                                     _pre_step_state, _print_report)

pytestmark = pytest.mark.gpu

D128 = dict(num_attention_heads=2, num_key_value_heads=1)   # 2 heads x 128 over a hidden size of 256
CONFIGS = {
    "qwen2-d64": dict(model="debug-qwen2", B=2, S=256, overrides={}),
    "qwen2-d64-tied": dict(model="debug-qwen2", B=2, S=256, overrides=dict(tie_word_embeddings=True)),
    "qwen2-d128": dict(model="debug-qwen2", B=2, S=256, overrides=D128),
    "qwen2-d128-tied": dict(model="debug-qwen2", B=2, S=256, overrides=dict(tie_word_embeddings=True, **D128)),
}


def _randomise_biases(eng, scale=0.02):
    """Zero-initialised biases would make the forward add vacuous: give them values (the flat views in place).  They
    stay below the projections' outputs (about 0.3): a k bias that dominated k would make the q gradient a
    cancellation (softmax ignores a shift shared by all keys) whose bf16 noise no reference could judge."""
    g = torch.Generator(device="cuda").manual_seed(3)
    with torch.no_grad():
        for n, p in eng.model.named_parameters():
            if n.endswith(".bias"):
                p.copy_(torch.randn(p.shape, device="cuda", generator=g) * scale)


def _split_k_bias(grads, ref_grads, bf16_grads, limit=GRAD_CEILING):
    """The k bias gradient nearly cancels: a k bias shifts all the scores of a query by the same amount, which softmax
    ignores, and only RoPE breaks that.  Its own relative error therefore measures the bf16 noise of dk, not the bias
    path.  Check it against the size of the layer's whole q|k|v bias gradient, and hand back the other gradients for
    the per-parameter check."""
    ks = [n for n in ref_grads if n.endswith("k_proj.bias")]
    for n in ks:
        whole = torch.cat([ref_grads[n.replace("k_proj", m)] for m in ("q_proj", "k_proj", "v_proj")])
        err = ((grads[n] - ref_grads[n]).norm() / whole.norm()).item()
        assert err <= limit, (n, err)
    keep = [n for n in ref_grads if n not in ks]
    return {n: ref_grads[n] for n in keep}, (None if bf16_grads is None else {n: bf16_grads[n] for n in keep})


@pytest.mark.parametrize("case", list(CONFIGS))
def test_qwen2_step_matches_fp32_reference(case, monkeypatch):
    cfg = CONFIGS[case]
    report, worst = [], 0.0
    with _engine(monkeypatch, cfg) as eng:
        config = eng.config
        assert config.qkv_bias and config.head_dim == (128 if "d128" in case else 64)
        _randomise_biases(eng)
        rec = _capture_buckets(eng)
        for step in (1, 2, 3):
            batch = eng.synthetic_batch(seed=step - 1)
            weights = {n: p.detach().clone() for n, p in eng.model.named_parameters()}
            assert sum(n.endswith(".bias") for n in weights) == 3 * config.num_hidden_layers
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
            ref_grads, bf16_grads = _split_k_bias(grads, ref_grads, bf16_grads)
            worst = max(worst, _check_grads(f"s{step}", grads, ref_grads, bf16_grads, report))
            _check_update(eng, rec, pre, step, lr)
    _print_report(f"{case}: per-parameter gradient error (worst ratio {worst:.2f})", report)


def test_qwen2_packed_step_matches_fp32_reference(monkeypatch):
    from distributed_training_guide_b200.engine import TrainEngine

    B, S = 2, 512
    eng = TrainEngine.create("debug-qwen2", parallelism="single", batch_size=B, seq_length=S, lr=5e-3, device="cuda",
                             document_masking=True)
    try:
        _randomise_biases(eng)
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
    _print_report("qwen2 packed step", report)


def test_qwen2_fp8_step_trains_the_biases(monkeypatch):
    """--fp8: the q|k|v GEMM runs in fp8 with the bias in its epilogue; the loss stays near the fp32 model's and the
    bias gradients (summed from the bf16 output gradient) are close to fp32's."""
    from distributed_training_guide_b200.engine import TrainEngine

    eng = TrainEngine.create("debug-qwen2", parallelism="single", batch_size=2, seq_length=256, lr=5e-3,
                             device="cuda", fp8=True)
    try:
        _randomise_biases(eng)
        weights = {n: p.detach().clone() for n, p in eng.model.named_parameters()}
        rec = _capture_buckets(eng)
        batch = eng.synthetic_batch(seed=0)
        loss = float(eng.step(batch))
        grads = _engine_grads(eng, rec)
        after = {n: p.detach().clone() for n, p in eng.model.named_parameters() if n.endswith(".bias")}
    finally:
        eng.close()
    (l32,), g32 = _plain_model_grads(eng.config, {n: w.float() for n, w in weights.items()}, [batch], torch.float32,
                                     monkeypatch)
    assert math.isfinite(loss) and abs(loss - l32) < 5e-2, (loss, l32)
    g32, _ = _split_k_bias(grads, g32, None, limit=0.2)
    for n, want in g32.items():
        if n.endswith(".bias"):
            err = ((grads[n] - want).norm() / want.norm()).item()
            assert err < 0.2, (n, err)   # fp8 e4m3 activations and weights: 3 mantissa bits
            assert not torch.equal(after[n], weights[n]), n


def test_qwen2_max_grad_norm_step(monkeypatch):
    from distributed_training_guide_b200.engine import TrainEngine

    eng = TrainEngine.create("debug-qwen2", parallelism="single", batch_size=2, seq_length=256, lr=5e-3,
                             device="cuda", max_grad_norm=1e-3)
    try:
        _randomise_biases(eng)
        weights = {n: p.detach().clone() for n, p in eng.model.named_parameters()}
        rec = _capture_buckets(eng)
        batch = eng.synthetic_batch(seed=0)
        eng.step(batch)
        norm = float(eng.grad_norm())
        grads = _engine_grads(eng, rec)
    finally:
        eng.close()
    own = math.sqrt(sum(float(g.double().pow(2).sum()) for g in grads.values()))
    assert abs(norm - own) <= 2e-6 * own, (norm, own)
    (_,), g32 = _plain_model_grads(eng.config, {n: w.float() for n, w in weights.items()}, [batch], torch.float32,
                                   monkeypatch)
    params = [torch.nn.Parameter(torch.zeros_like(g)) for g in g32.values()]
    for p, g in zip(params, g32.values()):
        p.grad = g.clone()
    ref_norm = float(torch.nn.utils.clip_grad_norm_(params, 1e-3))
    assert abs(norm - ref_norm) <= 2e-2 * ref_norm, (norm, ref_norm)


CHAPTER_ARGS = ["-d", "synthetic", "-m", "debug-qwen2", "-s", "256", "-b", "2", "--num-samples", "32", "--log-freq",
                "1", "-e", "exp", "--lr", "1e-3", "--max-steps", "4"]


def _losses(recs):
    return [r["running_loss"] for r in sorted(recs, key=lambda r: r["global_step"])]


def test_chapter01_qwen2_on_gpu(tmp_path):
    recs, _ = _run(ROOT / "01-single-gpu" / "train_llm.py", CHAPTER_ARGS + ["--save-dir", str(tmp_path)])
    assert len(recs) == 4 and all(r["tokens_per_s"] > 0 for r in recs)
    assert all(0 < l < 20 and math.isfinite(l) for l in _losses(recs))


@pytest.mark.multigpu
@pytest.mark.parametrize("chapter", ["02-distributed-data-parallel", "04-fully-sharded-data-parallel",
                                     "06-tensor-parallel"])
def test_distributed_chapters_qwen2_match_single_gpu(tmp_path, chapter):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    single, _ = _run(ROOT / "01-single-gpu" / "train_llm.py", CHAPTER_ARGS + ["--save-dir", str(tmp_path / "one")])
    recs, _ = _run(ROOT / chapter / "train_llm.py", CHAPTER_ARGS + ["--save-dir", str(tmp_path / "many")], nproc=2)
    a, b = _losses(single), _losses(recs)
    assert abs(a[0] - b[0]) < 5e-2, (a, b)
    assert all(math.isfinite(x) and x < a[0] + 0.5 for x in b), (a, b)
