"""Gradient clipping by global norm on the CPU: the reference path (``FlatAdamW`` / ``ref.clip_coefficient``) against
``torch.nn.utils.clip_grad_norm_`` + ``torch.optim.AdamW``, DDP over gloo against one process, the
``--max-grad-norm`` flag, the engines that refuse it and the log record."""
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

from dist_utils import initial_weights, run_distributed, update_rel_err

ROOT = Path(__file__).resolve().parents[1]


# ------------------------------------------------------------------------------------------------------------------
# the coefficient
# ------------------------------------------------------------------------------------------------------------------
def test_clip_coefficient_matches_torch():
    from distributed_training_guide_b200.ops import reference as ref

    for norm, max_norm in [(3.0, 1.0), (0.5, 1.0), (1.0, 1.0), (0.0, 0.1), (1e30, 1.0), (2.5, 1e30)]:
        g = torch.tensor([norm], dtype=torch.float32)
        g.grad = torch.tensor([norm], dtype=torch.float32)
        got_norm = torch.nn.utils.clip_grad_norm_([g], max_norm)
        want = g.grad / norm if norm else torch.ones(1)
        coef = ref.clip_coefficient(torch.tensor(norm, dtype=torch.float32), max_norm)
        assert float(got_norm) == pytest.approx(norm)
        if norm:
            assert float(coef) == pytest.approx(float(want), rel=1e-6), (norm, max_norm)
        assert float(coef) <= 1.0
    # not special-cased: the step goes non-finite, as torch's does
    assert torch.isnan(ref.clip_coefficient(torch.tensor(float("nan")), 1.0))
    assert float(ref.clip_coefficient(torch.tensor(float("inf")), 1.0)) == 0.0


# ------------------------------------------------------------------------------------------------------------------
# the CPU engine against torch, fp32 debug-llama
# ------------------------------------------------------------------------------------------------------------------
def _fp32_engine(monkeypatch, max_norm):
    from distributed_training_guide_b200.engine import TrainEngine
    from distributed_training_guide_b200.parallel import strategies

    monkeypatch.setattr(strategies.SingleDevice, "dtype", lambda self: torch.float32)
    torch.manual_seed(0)
    return TrainEngine.create("debug-llama", parallelism="single", batch_size=2, seq_length=32, device="cpu", lr=1e-2,
                              max_grad_norm=max_norm)


def _torch_twin(eng):
    from distributed_training_guide_b200.models.llama import build_llama

    model = build_llama(eng.config, dtype=torch.float32, device="cpu", init=False)
    with torch.no_grad():
        for (n, p), (n2, q) in zip(model.named_parameters(), eng.model.named_parameters()):
            assert n == n2
            p.copy_(q)
    opt = torch.optim.AdamW(model.parameters(), lr=1e-2, foreach=False)
    return model, opt


def _batches(eng, step, accum):
    out = []
    for k in range(accum):
        g = torch.Generator().manual_seed(100 * step + k)
        ids = torch.randint(0, eng.config.vocab_size, (2, 32), generator=g)
        out.append({"input_ids": ids, "labels": ids.clone()})
    return out


@pytest.mark.parametrize("accum", [1, 2])
@pytest.mark.parametrize("max_norm", [1e-2, 1e6], ids=["clips", "no-op"])
def test_cpu_engine_matches_clip_grad_norm_and_adamw(monkeypatch, max_norm, accum):
    eng = _fp32_engine(monkeypatch, max_norm)
    model, opt = _torch_twin(eng)
    s = eng.strategy
    for step in range(3):
        lr = eng.optimizer.lr
        for pg in opt.param_groups:
            pg["lr"] = lr
        batches = _batches(eng, step, accum)
        for k, b in enumerate(batches):
            out = eng.model(**s.prepare_batch(dict(b)))
            with s.grad_sync(eng.model, enabled=k == accum - 1):
                s.backward(eng.model, out.loss / accum)
            (model(**b).loss / accum).backward()
        eng.optimizer.step()
        eng.lr_scheduler.step()
        eng.optimizer.zero_grad()
        want_norm = torch.nn.utils.clip_grad_norm_(model.parameters(), max_norm)
        opt.step()
        opt.zero_grad()
        got_norm = eng.grad_norm()
        assert got_norm.dtype == torch.float32
        assert float(got_norm) == pytest.approx(float(want_norm), rel=1e-5), step
        assert (float(want_norm) > max_norm) == (max_norm < 1), "the case does not exercise what it is named after"
        # AdamW's update barely depends on the gradient's scale, its moments do: they show a wrong coefficient
        twin = dict(model.named_parameters())
        for g in eng.optimizer.flat_groups:
            st = eng.optimizer.state[g.param]
            for n, o, p in zip(g.names, g.offsets, g.params):
                ts = opt.state[twin[n]]
                for key in ("exp_avg", "exp_avg_sq"):
                    got = st[key][o:o + p.numel()].view(p.shape)
                    scale = float(ts[key].abs().max())
                    torch.testing.assert_close(got, ts[key], rtol=1e-4, atol=1e-5 * scale,
                                               msg=lambda m: f"step {step} {n} {key}: {m}")
                # a gradient near zero can flip the sign of one lr-sized step between two fp32 orders of summation
                torch.testing.assert_close(p, twin[n], rtol=1e-5, atol=1e-5, msg=lambda m: f"step {step} {n}: {m}")


def test_norm_covers_each_parameter_once_and_no_padding():
    """The flat groups' padding (between parameters and at the tail) never reaches the norm; a tied embedding is
    one parameter, counted once."""
    from distributed_training_guide_b200.engine import TrainEngine

    eng = TrainEngine.create("debug-gpt2", parallelism="single", batch_size=2, seq_length=32, device="cpu",
                             max_grad_norm=1.0)
    opt = eng.optimizer
    for g in opt.flat_groups:
        g.grad.fill_(float("nan"))
        for p in g.params:
            p.grad.fill_(0.5)
    params = {id(p): p for p in eng.model.parameters()}
    n_elems = sum(p.numel() for p in params.values())
    assert any(g.padded_numel > sum(p.numel() for p in g.params) for g in opt.flat_groups), "no padding to test"
    assert float(opt.global_grad_norm()) == pytest.approx(0.5 * n_elems ** 0.5, rel=1e-6)


def test_gpt2_single_engine_clips_on_cpu():
    from distributed_training_guide_b200.engine import TrainEngine

    eng = TrainEngine.create("debug-gpt2", parallelism="single", batch_size=2, seq_length=32, device="cpu",
                             max_grad_norm=0.5)
    eng.step(eng.synthetic_batch(seed=0, pinned=False))
    assert float(eng.grad_norm()) > 0.5
    assert TrainEngine.create("debug-gpt2", parallelism="single", device="cpu").grad_norm() is None


# ------------------------------------------------------------------------------------------------------------------
# DDP over gloo against one process on the global batch
# ------------------------------------------------------------------------------------------------------------------
MAX_NORM = 0.05  # well below the norm of debug-llama's gradients at init: every step clips


def _train(rank, world, parallelism, steps):
    from distributed_training_guide_b200.engine import TrainEngine

    torch.manual_seed(0)
    eng = TrainEngine.create("debug-llama", parallelism=parallelism, batch_size=2, seq_length=32, device="cpu",
                             lr=1e-3, max_grad_norm=MAX_NORM)
    norms = []
    for i in range(steps):
        eng.step(eng.synthetic_batch(seed=i, pinned=False))
        norms.append(float(eng.grad_norm()))
    return norms, {k: v.detach().float().clone() for k, v in eng.model.state_dict().items()}


def _single(steps, world):
    from distributed_training_guide_b200.engine import TrainEngine

    torch.manual_seed(0)
    eng = TrainEngine.create("debug-llama", parallelism="single", batch_size=2 * world, seq_length=32, device="cpu",
                             lr=1e-3, max_grad_norm=MAX_NORM)
    norms = []
    for i in range(steps):
        parts = [torch.randint(0, eng.config.vocab_size, (2, 32), generator=torch.Generator().manual_seed(1000 * i + r))
                 for r in range(world)]
        ids = torch.cat(parts)
        eng.step({"input_ids": ids, "labels": ids.clone()})
        norms.append(float(eng.grad_norm()))
    return norms, {k: v.detach().float().numpy() for k, v in eng.model.state_dict().items()}


@pytest.mark.parametrize("parallelism", ["ddp", "ddp_allreduce"])
def test_ddp_clipping_matches_single_process(parallelism):
    steps, world = 3, 2
    (n0, sd0), (n1, sd1) = run_distributed(_train, world=world, args=(parallelism, steps))
    ref_norms, ref_sd = _single(steps, world)
    assert n0 == n1, "ranks disagree on the norm"
    for k in sd0:
        assert np.array_equal(sd0[k], sd1[k]), k
    for i in range(steps):
        assert n0[i] > MAX_NORM
        assert n0[i] == pytest.approx(ref_norms[i], rel=2e-2), (i, n0[i], ref_norms[i])
    err = update_rel_err(initial_weights(), sd0, ref_sd)
    assert err < 0.1, err


# ------------------------------------------------------------------------------------------------------------------
# flag, refusals, log record
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("chapter", ["01-single-gpu", "02-distributed-data-parallel", "04-fully-sharded-data-parallel",
                                     "05-training-llama-405b", "06-tensor-parallel", "07-2d-parallel", "deepspeed"])
def test_max_grad_norm_flag_only_in_chapters_01_and_02(chapter):
    from distributed_training_guide_b200.utils.cli import get_parser

    base = ["-d", "synthetic", "-m", "debug-llama"]
    p = get_parser(chapter)
    assert p.parse_args(base).__dict__.get("max_grad_norm") is None
    if chapter in ("01-single-gpu", "02-distributed-data-parallel"):
        assert p.parse_args(base + ["--max-grad-norm", "1.0"]).max_grad_norm == 1.0
        for bad in ("0", "-1", "nan"):
            with pytest.raises(SystemExit):
                p.parse_args(base + ["--max-grad-norm", bad])
    else:
        with pytest.raises(SystemExit):
            p.parse_args(base + ["--max-grad-norm", "1.0"])


@pytest.mark.parametrize("parallelism", ["fsdp", "tp", "2d"])
def test_max_grad_norm_rejected_by_other_engines(parallelism):
    from distributed_training_guide_b200.engine import TrainEngine

    with pytest.raises(ValueError, match="single, ddp, ddp_allreduce"):
        TrainEngine.create("debug-llama", parallelism=parallelism, device="cpu", max_grad_norm=1.0)


@pytest.mark.parametrize("value", [0.0, -1.0])
def test_non_positive_max_grad_norm_rejected(value):
    from distributed_training_guide_b200.engine import TrainEngine

    with pytest.raises(ValueError, match="> 0"):
        TrainEngine.create("debug-llama", parallelism="single", device="cpu", max_grad_norm=value)


def _chapter01(tmp_path, extra):
    script = ROOT / "01-single-gpu" / "train_llm.py"
    cmd = [sys.executable, str(script), "-d", "synthetic", "-m", "debug-llama", "-s", "32", "-b", "2",
           "--num-samples", "32", "--log-freq", "1", "--max-steps", "2", "--lr", "1e-3", "--device", "cpu",
           "--save-dir", str(tmp_path), *extra]
    r = subprocess.run(cmd, capture_output=True, text=True, cwd=str(script.parent), timeout=300)
    assert r.returncode == 0, (r.stdout + r.stderr)[-3000:]
    return [eval(line.split("INFO:", 1)[1]) for line in r.stderr.splitlines() if "INFO:{" in line]


def test_log_record_has_grad_norm_only_with_the_flag(tmp_path):
    on = _chapter01(tmp_path / "on", ["--max-grad-norm", "0.5"])
    off = _chapter01(tmp_path / "off", [])
    assert [r["global_step"] for r in on] == [1, 2] and [r["global_step"] for r in off] == [1, 2]
    assert all(np.isfinite(r["grad_norm"]) and r["grad_norm"] > 0 for r in on)
    assert all("grad_norm" not in r for r in off)
    assert set(on[0]) - set(off[0]) == {"grad_norm"}
