"""FP8 linears on the CPU: the reference quantisation (the definition the cast kernels are tested against bit for
bit), the op's backward, the ``--fp8`` flag and engine plumbing, DDP over gloo, checkpoints and resume."""
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

from dist_utils import run_distributed
from distributed_training_guide_b200 import ops
from distributed_training_guide_b200.ops import reference as ref

ROOT = Path(__file__).resolve().parent.parent
E4M3, E5M2 = torch.float8_e4m3fn, torch.float8_e5m2


# ------------------------------------------------------------------------------------------------------------------
# reference quantisation
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype,fmax", [(E4M3, 448.0), (E5M2, 57344.0)], ids=["e4m3", "e5m2"])
def test_quantize_maps_amax_to_fp8_max_and_saturates(dtype, fmax):
    x = torch.tensor([[3.0, -1.5, 0.25, 0.0], [-3.0, 1e-30, 2.0, 1.0]])
    t8, scale_inv = ref.fp8_quantize(x, dtype)
    assert t8.dtype == dtype
    assert t8.float()[0, 0] == fmax and t8.float()[1, 0] == -fmax
    assert scale_inv.dtype == torch.float32 and scale_inv.shape == (1,)
    assert scale_inv.item() == pytest.approx(3.0 / fmax, rel=1e-7)
    # an amax below the true max (a stale scale) saturates at +-FP8_MAX instead of giving NaN / Inf
    t8s, _ = ref.fp8_quantize(x, dtype, amax=torch.tensor([0.5]))
    assert t8s.float().abs().max().item() == fmax
    assert torch.isfinite(t8s.float()).all()
    assert t8s.float()[0, 0] == fmax and t8s.float()[0, 1] == -fmax


def test_quantize_zero_tensor_has_unit_scale():
    t8, scale_inv = ref.fp8_quantize(torch.zeros(3, 5), E4M3)
    assert scale_inv.item() == 1.0
    assert torch.equal(t8.view(torch.uint8), torch.zeros(3, 5, dtype=torch.uint8))


@pytest.mark.parametrize("bad", [float("inf"), float("-inf"), float("nan")])
@pytest.mark.parametrize("dtype", [E4M3, E5M2], ids=["e4m3", "e5m2"])
def test_quantize_nonfinite_input_stays_nonfinite(bad, dtype):
    x = torch.randn(4, 8)
    x[2, 3] = bad
    t8, scale_inv = ref.fp8_quantize(x, dtype)
    assert not bool(torch.isfinite(t8.float()).all())
    deq = ref.fp8_gemm(t8, scale_inv, ref.fp8_quantize(torch.randn(6, 8), E4M3)[0], torch.ones(1))
    assert not bool(torch.isfinite(deq).all()), "a non-finite input must reach the GEMM output"


BF16_MIN_SUBNORMAL = 2.0 ** -133


@pytest.mark.parametrize("amax", [1e-37, 1e-36, 1e-34, BF16_MIN_SUBNORMAL], ids=["1e-37", "1e-36", "1e-34", "min"])
@pytest.mark.parametrize("dtype", [E4M3, E5M2], ids=["e4m3", "e5m2"])
def test_quantize_tiny_amax_stays_finite(dtype, amax):
    """FP8_MAX / amax overflows fp32 below amax = FP8_MAX / FLT_MAX (1.3e-36 for e4m3, 1.7e-34 for e5m2): the scale is
    clamped to FLT_MAX, so zeros stay zero and every element still dequantises to within fp8 rounding of x."""
    top = torch.tensor(amax, dtype=torch.bfloat16).float().item()
    x = torch.tensor([[0.0, top, -top, 0.5 * top], [-0.0, 0.3 * top, -0.7 * top, 0.0]]).to(torch.bfloat16)
    t8, scale_inv = ref.fp8_quantize(x, dtype)
    q = t8.float()
    assert not bool(torch.isnan(q).any()), q
    assert (q[x == 0] == 0).all()
    assert 0 < scale_inv.item() < float("inf")
    u, sub = (2.0 ** -4, 2.0 ** -9) if dtype == E4M3 else (2.0 ** -3, 2.0 ** -16)   # unit roundoff, least subnormal
    xd, deq = x.double(), q.double() * scale_inv.double()
    tol = (u + 2.0 ** -22) * xd.abs() + 0.5 * sub * scale_inv.double()
    assert ((deq - xd).abs() <= tol).all(), (deq, xd)


def test_quantize_rounds_to_nearest_even():
    # with amax 448 the scale is exactly 1: 17 and 19 lie halfway between e4m3 neighbours (16, 18, 20)
    x = torch.tensor([[448.0, 17.0, 19.0, -17.0]])
    t8, _ = ref.fp8_quantize(x, E4M3)
    assert t8.float().tolist() == [[448.0, 16.0, 20.0, -16.0]]


# ------------------------------------------------------------------------------------------------------------------
# the op
# ------------------------------------------------------------------------------------------------------------------
def test_fp8_linear_forward_and_backward_follow_the_recipe():
    """Forward quantises x and W to e4m3, backward quantises dy to e5m2; every product is the fp32 product of the
    dequantised operands, rounded to bf16."""
    g = torch.Generator().manual_seed(0)
    x = torch.randn(2, 16, 64, generator=g).to(torch.bfloat16).requires_grad_()
    w = (0.05 * torch.randn(48, 64, generator=g)).to(torch.bfloat16).requires_grad_()
    dy = (1e-3 * torch.randn(2, 16, 48, generator=g)).to(torch.bfloat16)
    y = ops.linear(x, w, fp8=True)
    y.backward(dy)

    x8, sx = ref.fp8_quantize(x.detach().reshape(32, 64), E4M3)
    w8, sw = ref.fp8_quantize(w.detach(), E4M3)
    dy8, sdy = ref.fp8_quantize(dy.reshape(32, 48), E5M2)
    deq = lambda t8, s: t8.float() * s  # noqa: E731
    want_y = (deq(x8, sx) @ deq(w8, sw).t()).to(torch.bfloat16).view(2, 16, 48)
    want_dx = (deq(dy8, sdy) @ deq(w8, sw)).to(torch.bfloat16).view(2, 16, 64)
    want_dw = (deq(dy8, sdy).t() @ deq(x8, sx)).to(torch.bfloat16)
    for name, got, want in (("y", y, want_y), ("dx", x.grad, want_dx), ("dw", w.grad, want_dw)):
        assert torch.allclose(got.float(), want.float(), rtol=8e-3, atol=1e-6), name

    # dy in e4m3 would give a different dx: the backward really uses e5m2
    dy8_e4, sdy_e4 = ref.fp8_quantize(dy.reshape(32, 48), E4M3)
    other = (deq(dy8_e4, sdy_e4) @ deq(w8, sw)).to(torch.bfloat16).view(2, 16, 64)
    assert not torch.equal(other, want_dx)
    assert (x.grad.float() - want_dx.float()).abs().max() < (x.grad.float() - other.float()).abs().max()


def test_fp8_linear_writes_into_the_flat_gradient_view():
    """A weight carrying ``_dtg_grad`` gets its gradient written into that view (overwrite on first use, accumulate
    afterwards) and hands None to autograd."""
    g = torch.Generator().manual_seed(1)
    w = (0.05 * torch.randn(32, 64, generator=g)).to(torch.bfloat16)
    buf = torch.full((32 * 64 + 16,), 7.0, dtype=torch.bfloat16)
    w._dtg_grad = buf[8:8 + 32 * 64].view(32, 64)
    w._dtg_writes = 0
    x = torch.randn(16, 64, generator=g).to(torch.bfloat16)
    dy = torch.randn(16, 32, generator=g).to(torch.bfloat16)
    ops.linear(x.requires_grad_(), w.requires_grad_(), fp8=True).backward(dy)
    first = w._dtg_grad.clone()
    assert w.grad is None and w._dtg_writes == 1
    assert torch.equal(buf[:8], torch.full((8,), 7.0, dtype=torch.bfloat16))
    ops.linear(x, w, fp8=True).backward(dy)
    assert w._dtg_writes == 2
    assert torch.allclose(w._dtg_grad.float(), 2 * first.float(), rtol=1e-2)


# ------------------------------------------------------------------------------------------------------------------
# flag and engines
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("chapter", ["01-single-gpu", "02-distributed-data-parallel", "04-fully-sharded-data-parallel",
                                     "05-training-llama-405b", "06-tensor-parallel", "07-2d-parallel", "deepspeed"])
def test_fp8_flag_only_in_chapters_01_and_02(chapter):
    from distributed_training_guide_b200.utils.cli import get_parser

    base = ["-d", "synthetic", "-m", "debug-llama"]
    p = get_parser(chapter)
    assert p.parse_args(base).__dict__.get("fp8", False) is False
    if chapter in ("01-single-gpu", "02-distributed-data-parallel"):
        assert p.parse_args(base + ["--fp8"]).fp8 is True
    else:
        with pytest.raises(SystemExit):
            p.parse_args(base + ["--fp8"])


@pytest.mark.parametrize("parallelism", ["fsdp", "tp", "2d"])
def test_fp8_rejected_by_sharded_engines(parallelism):
    from distributed_training_guide_b200.engine import TrainEngine

    with pytest.raises(ValueError, match="single, ddp, ddp_allreduce"):
        TrainEngine.create("debug-llama", parallelism=parallelism, device="cpu", fp8=True)


def test_fp8_rejected_for_gpt2():
    from distributed_training_guide_b200.engine import TrainEngine

    with pytest.raises(ValueError, match="Llama"):
        TrainEngine.create("debug-gpt2", parallelism="single", device="cpu", fp8=True)


def test_fp8_is_off_by_default_and_routes_the_projections():
    from distributed_training_guide_b200.engine import TrainEngine

    calls = []
    real = ops.linear
    eng = TrainEngine.create("debug-llama", parallelism="single", batch_size=2, seq_length=32, device="cpu")
    assert eng.model.fp8 is False and not any(layer.fp8 for layer in eng.model.model.layers)
    eng_fp8 = TrainEngine.create("debug-llama", parallelism="single", batch_size=2, seq_length=32, device="cpu",
                                 fp8=True)
    assert all(layer.fp8 for layer in eng_fp8.model.model.layers)
    try:
        ops.linear = lambda *a, **k: (k.get("fp8") and calls.append(a[1].shape)) or real(*a, **k)
        eng.step(eng.synthetic_batch(seed=0, pinned=False))
        assert calls == []
        eng_fp8.step(eng_fp8.synthetic_batch(seed=0, pinned=False))
    finally:
        ops.linear = real
    assert len(calls) == 4 * eng_fp8.config.num_hidden_layers


# ------------------------------------------------------------------------------------------------------------------
# DDP, checkpoints, resume, the chapter script
# ------------------------------------------------------------------------------------------------------------------
def _ddp_fp8(rank, world, steps):
    from distributed_training_guide_b200.engine import TrainEngine

    torch.manual_seed(0)
    eng = TrainEngine.create("debug-llama", parallelism="ddp", batch_size=2, seq_length=32, device="cpu", lr=1e-3,
                             fp8=True)
    assert eng.model.fp8
    losses = [float(eng.step(eng.synthetic_batch(seed=i, pinned=False))) for i in range(steps)]
    return losses, {k: v.detach().float().clone() for k, v in eng.model.state_dict().items()}


def test_fp8_ddp_matches_single_process():
    from distributed_training_guide_b200.engine import TrainEngine

    steps, world = 3, 2
    (l0, sd0), (l1, sd1) = run_distributed(_ddp_fp8, world=world, args=(steps,))
    torch.manual_seed(0)
    eng = TrainEngine.create("debug-llama", parallelism="single", batch_size=2, seq_length=32, device="cpu", lr=1e-3,
                             fp8=True)
    want = []
    for i in range(steps):
        parts = [torch.randint(0, eng.config.vocab_size, (2, 32), generator=torch.Generator().manual_seed(1000 * i + r))
                 for r in range(world)]
        ids = torch.cat(parts)
        want.append(float(eng.step({"input_ids": ids, "labels": ids.clone()})))
    sd = {k: v.detach().float().numpy() for k, v in eng.model.state_dict().items()}
    for k in sd0:
        assert np.array_equal(sd0[k], sd1[k]), f"replicas diverged: {k}"
    for i in range(steps):
        assert abs(0.5 * (l0[i] + l1[i]) - want[i]) < 2e-2, (i, l0[i], l1[i], want[i])
    for k in sd0:
        assert np.abs(sd0[k] - sd[k]).max() < 2e-2, k


def _run(tmp, fp8, steps_before, steps_after=0, resume=False):
    from distributed_training_guide_b200.engine import TrainEngine

    def make():
        torch.manual_seed(0)
        return TrainEngine.create("debug-llama", parallelism="single", batch_size=2, seq_length=32, device="cpu",
                                  lr=1e-2, fp8=fp8)

    eng = make()
    batches = [eng.synthetic_batch(seed=i, pinned=False) for i in range(steps_before + steps_after)]
    losses = [float(eng.step(b)) for b in batches[:steps_before]]
    if tmp is not None:
        tmp.mkdir(parents=True, exist_ok=True)
        eng.strategy.save_checkpoint(tmp, eng.model, eng.optimizer, eng.lr_scheduler,
                                     {"epoch": 0, "global_step": steps_before, "epoch_step": steps_before,
                                      "running_loss": 0.0})
    if resume:
        eng = make()
        st = eng.strategy.load_checkpoint(tmp, eng.model, eng.optimizer, eng.lr_scheduler)
        assert st["global_step"] == steps_before
    losses += [float(eng.step(b)) for b in batches[steps_before:]]
    return losses, eng


def test_fp8_checkpoint_has_the_bf16_layout(tmp_path):
    _run(tmp_path / "bf16", False, 2)
    _run(tmp_path / "fp8", True, 2)
    for name in ("model.pt", "optimizer.pt"):
        a = torch.load(tmp_path / "bf16" / name, weights_only=False)
        b = torch.load(tmp_path / "fp8" / name, weights_only=False)
        flat = lambda d, p="": {f"{p}{k}": v for k, v in d.items()} if isinstance(d, dict) else {p: d}  # noqa: E731
        fa, fb = flat(a), flat(b)
        assert sorted(fa) == sorted(fb), name
        for k in fa:
            if isinstance(fa[k], torch.Tensor):
                assert fa[k].dtype == fb[k].dtype and fa[k].shape == fb[k].shape, (name, k)


def test_fp8_resume_reproduces_the_uninterrupted_run(tmp_path):
    straight, _ = _run(None, True, 4)
    resumed, _ = _run(tmp_path / "exp", True, 2, 2, resume=True)
    assert straight == resumed, (straight, resumed)


def test_chapter01_trains_with_fp8_on_cpu(tmp_path):
    script = ROOT / "01-single-gpu" / "train_llm.py"
    cmd = [sys.executable, str(script), "-d", "synthetic", "-m", "debug-llama", "-s", "32", "-b", "2",
           "--num-samples", "32", "--log-freq", "1", "--max-steps", "3", "--lr", "1e-3", "--device", "cpu", "--fp8",
           "--save-dir", str(tmp_path)]
    r = subprocess.run(cmd, capture_output=True, text=True, cwd=str(script.parent), timeout=300)
    assert r.returncode == 0, (r.stdout + r.stderr)[-3000:]
    recs = [eval(line.split("INFO:", 1)[1]) for line in r.stderr.splitlines() if "INFO:{" in line]
    assert [rec["global_step"] for rec in recs] == [1, 2, 3]
    assert all(0 < rec["running_loss"] < 20 for rec in recs)
