"""FP8 training of the decoder-layer projections: amax and cast-transpose kernels bit for bit against the reference
quantisation, the fp8 wgmma GEMM against the fp32 product of its dequantised operands (with ``torch._scaled_mm`` on the
same operands as the yardstick), and the fp8 training step against an fp32 model, relative to the error of the same
model with PyTorch fp8 GEMMs.
"""
import contextlib
import gc
import math

import pytest
import torch

from distributed_training_guide_b200 import _ext, ops
from distributed_training_guide_b200 import engine as engine_mod
from distributed_training_guide_b200.models.llama import build_llama
from distributed_training_guide_b200.ops import reference as ref
from test_gpu_step_reference import (CONFIGS, GRAD_SLACK, LOSS_FACTOR, LOSS_SLACK, LR,
                                     _capture_buckets, _check_order, _check_update, _engine_grads, _fp32_matmuls,
                                     _plain_model_grads, _pre_step_state, _rel)

pytestmark = pytest.mark.gpu

E4M3, E5M2 = torch.float8_e4m3fn, torch.float8_e5m2


def _C():
    return _ext.load(True)


def _bits(t):
    return t.view(torch.uint8)


def _same_bits_nan_aware(got, want):
    """Bit-identical, except that a NaN may carry either sign (the CPU makes -NaN of Inf * 0, the GPU +NaN)."""
    gn, wn = torch.isnan(got.float()), torch.isnan(want.float())
    assert torch.equal(gn, wn), f"NaN positions differ: {int((gn != wn).sum())}"
    gb, wb = _bits(got)[~gn], _bits(want)[~wn]
    bad = int((gb != wb).sum())
    assert bad == 0, f"{bad} of {gb.numel()} fp8 values differ"


def _input(shape, kind, seed=0, std=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(*shape, device="cuda", generator=g) * std
    if kind == "zeros":
        x.zero_()
    elif kind == "inf":
        x[shape[0] // 3, shape[1] // 2] = float("inf")
    elif kind == "wide":   # 1e-8 .. 1e4: subnormals of both formats and saturation-free tails
        x = x * torch.exp(6 * torch.randn(*shape, device="cuda", generator=g))
    elif kind == "tiny":   # amax ~ 4e-37, below FP8_MAX / FLT_MAX of both formats, with zeros
        x = x * 1e-37
        x[:, ::5] = 0
    x = x.to(torch.bfloat16)
    # views of a larger buffer: "strided" keeps the 16-byte vector path (ld > C, ld % 8 == 0, aligned base),
    # "misaligned" (base 2 bytes past a 16-byte boundary) and "odd-ld" (ld = C + 3) take the scalar path
    pad = {"strided": (8, 16), "misaligned": (1, 7), "odd-ld": (0, 3)}.get(kind)
    if pad is not None:
        buf = torch.full((shape[0], pad[0] + shape[1] + pad[1]), float("nan"), device="cuda", dtype=torch.bfloat16)
        view = buf[:, pad[0]:pad[0] + shape[1]]
        view.copy_(x)
        x = view
    return x


# ------------------------------------------------------------------------------------------------------------------
# amax and cast-transpose
# ------------------------------------------------------------------------------------------------------------------
CAST_SHAPES = [(1000, 4104), (4096, 4096), (256, 11008), (7, 33), (129, 130)]
CAST_KINDS = ["normal", "wide", "zeros", "inf", "tiny", "strided", "misaligned", "odd-ld"]


@pytest.mark.parametrize("shape", CAST_SHAPES)
@pytest.mark.parametrize("kind", CAST_KINDS)
def test_amax_exact(shape, kind):
    x = _input(shape, kind)
    got = _C().fp8_amax(x)
    assert got.dtype == torch.float32 and got.shape == (1,)
    assert torch.equal(got, x.float().abs().max().reshape(1)), (got.item(), x.float().abs().max().item())


def test_amax_strided_view():
    base = _input((512, 1000), "wide", seed=3)
    for view in (base[:, 8:1000], base[:, 3:901], base[100:300, :512]):
        assert torch.equal(_C().fp8_amax(view), view.float().abs().max().reshape(1))


@pytest.mark.parametrize("shape", CAST_SHAPES)
@pytest.mark.parametrize("kind", CAST_KINDS)
@pytest.mark.parametrize("dtype", [E4M3, E5M2], ids=["e4m3", "e5m2"])
def test_cast_transpose_exact(shape, kind, dtype):
    x = _input(shape, kind, seed=1)
    amax = _C().fp8_amax(x)
    x8, x8t, scale_inv = _C().fp8_cast_transpose(x, amax, dtype == E5M2, True, True)
    want8, want_si = ref.fp8_quantize(x.cpu(), dtype)   # a view is gathered into a contiguous copy first
    if kind != "inf":
        assert not bool(torch.isnan(x8.float()).any()), "a finite input quantised to NaN"
    if kind == "tiny":
        assert bool((x8.float()[x == 0] == 0).all()), "a zero did not stay zero"
    assert x8.dtype == dtype and x8.shape == shape and x8t.shape == shape[::-1]
    _same_bits_nan_aware(x8.cpu(), want8)
    assert torch.equal(_bits(x8t), _bits(x8).t()), "the transposed copy is not the transpose of the row-major copy"
    assert torch.equal(scale_inv.cpu(), want_si), (scale_inv.item(), want_si.item())
    if kind == "zeros":
        assert scale_inv.item() == 1.0
    if kind == "inf":
        assert not bool(torch.isfinite(x8.float()).all()), "an Inf in the input must not quantise to finite values"
        assert not math.isfinite(scale_inv.item())
    # saturation: values scaled past FP8_MAX (here none are, amax maps to FP8_MAX exactly) never exceed it
    finite = x8.float()[torch.isfinite(x8.float())]
    assert finite.abs().max().item() <= torch.finfo(dtype).max


@pytest.mark.parametrize("layout", ["rowwise", "transposed"])
def test_cast_single_layout(layout):
    x = _input((1000, 4104), "normal", seed=2)
    amax = _C().fp8_amax(x)
    x8, x8t, _ = _C().fp8_cast_transpose(x, amax, False, layout == "rowwise", layout == "transposed")
    want8, _ = ref.fp8_quantize(x.cpu(), E4M3)
    if layout == "rowwise":
        assert x8t is None and torch.equal(_bits(x8.cpu()), _bits(want8))
    else:
        assert x8 is None and torch.equal(_bits(x8t.cpu()), _bits(want8).t())


def test_cast_saturates_with_stale_amax():
    """An amax below the true max (as any scale other than the current one would give) saturates at FP8_MAX."""
    x = _input((256, 512), "normal", seed=4)
    for dtype in (E4M3, E5M2):
        amax = (x.float().abs().max() / 4).reshape(1)
        x8, _, _ = _C().fp8_cast_transpose(x, amax, dtype == E5M2, True, False)
        fmax = torch.finfo(dtype).max
        assert x8.float().abs().max().item() == fmax
        want = (x.float() * (torch.full_like(amax, fmax) / amax)).clamp(-fmax, fmax).to(dtype)
        assert torch.equal(_bits(x8), _bits(want))


# ------------------------------------------------------------------------------------------------------------------
# fp8 GEMM
# ------------------------------------------------------------------------------------------------------------------
# (M, N, K, A format): Llama-2-7B projections at T = 4096; dgrad A = dY, wgrad A = dY^T (e5m2)
GEMM_SHAPES = {
    "fwd-qkv": (4096, 12288, 4096, E4M3),
    "fwd-o": (4096, 4096, 4096, E4M3),
    "fwd-gate_up": (4096, 22016, 4096, E4M3),
    "fwd-down-K11008": (4096, 4096, 11008, E4M3),
    "dgrad-qkv": (4096, 4096, 12288, E5M2),
    "dgrad-down": (4096, 11008, 4096, E5M2),
    "wgrad-gate_up-T4096": (22016, 4096, 4096, E5M2),
    "wgrad-down-T16384": (4096, 11008, 16384, E5M2),
    "wgrad-o-T16384": (4096, 4096, 16384, E5M2),
    "odd-e4m3": (1040, 1200, 1040, E4M3),
    "odd-e5m2": (1040, 1200, 1040, E5M2),
}
TILE_M, TILE_N = 128, 256
# The kernel accumulates like cuBLASLt's fast-accumulation fp8 GEMM: measured worst-tile errors equal
# ``_scaled_mm(use_fast_accum=True)``'s to four digits on every shape (1.7e-3 at K 1040 to 3.3e-3 at K 16384, where the
# split-accumulator mode stays at 1.7e-3, the bf16 rounding of the output).
GEMM_FACTOR, GEMM_SLACK = 1.1, 2e-4


def _worst_tile(got, want):
    """Largest relative L2 error over the 128 x 256 output tiles."""
    M, N = want.shape
    d, w = (got.float() - want).double(), want.double()
    mt, nt = -(-M // TILE_M), -(-N // TILE_N)
    pad = lambda t: torch.nn.functional.pad(t, (0, nt * TILE_N - N, 0, mt * TILE_M - M))  # noqa: E731
    dn = pad(d).view(mt, TILE_M, nt, TILE_N).square().sum((1, 3)).sqrt()
    wn = pad(w).view(mt, TILE_M, nt, TILE_N).square().sum((1, 3)).sqrt()
    return (dn / wn.clamp_min(1e-30)).max().item()


def _operands(M, N, K, a_fmt, seed=0):
    a8, _, sa = ops.fp8_cast(_input((M, K), "normal", seed=seed, std=0.7), a_fmt, transposed=False)
    b8, _, sb = ops.fp8_cast(_input((N, K), "normal", seed=seed + 1, std=0.02), E4M3, transposed=False)
    return a8, sa, b8, sb


def _dequant_product(a8, sa, b8, sb):
    with _fp32_matmuls():
        return ref.fp8_gemm(a8, sa, b8, sb)


def _scaled_mm(a8, sa, b8, sb, fast):
    return torch._scaled_mm(a8, b8.t(), scale_a=sa, scale_b=sb, out_dtype=torch.bfloat16, use_fast_accum=fast)


@pytest.mark.parametrize("variant", [1, 2])
@pytest.mark.parametrize("case", list(GEMM_SHAPES))
def test_gemm_fp8_accuracy(case, variant):
    M, N, K, a_fmt = GEMM_SHAPES[case]
    a8, sa, b8, sb = _operands(M, N, K, a_fmt)
    assert sa.item() != 1.0 and sb.item() != 1.0
    want = _dequant_product(a8, sa, b8, sb)
    out = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
    _C().gemm_fp8(a8, b8, out, sa, sb, False, variant)
    out2 = torch.empty_like(out)
    _C().gemm_fp8(a8, b8, out2, sa, sb, False, variant)
    assert torch.equal(out, out2), "two calls on the same operands differ"
    err = _worst_tile(out, want)
    fast = _worst_tile(_scaled_mm(a8, sa, b8, sb, True), want)
    slow = _worst_tile(_scaled_mm(a8, sa, b8, sb, False), want)
    print(f"\n{case} variant {variant}: worst-tile rel err kernel {err:.3e}  _scaled_mm fast {fast:.3e}  "
          f"split {slow:.3e}")
    assert err <= GEMM_FACTOR * fast + GEMM_SLACK, (err, fast, slow)


@pytest.mark.parametrize("variant", [1, 2])
@pytest.mark.parametrize("case", ["odd-e5m2", "wgrad-gate_up-T4096"])
def test_gemm_fp8_accumulate_into_strided_view(case, variant):
    """Accumulate mode into a view of a larger buffer (a flat-gradient slice): C = old + product in fp32, and not
    one element outside the view changes."""
    M, N, K, a_fmt = GEMM_SHAPES[case]
    a8, sa, b8, sb = _operands(M, N, K, a_fmt, seed=5)
    g = torch.Generator(device="cuda").manual_seed(9)
    buf = (torch.randn(M + 48, N + 64, device="cuda", generator=g) * 0.05).to(torch.bfloat16)
    before = buf.clone()
    view = buf[16:16 + M, 32:32 + N]
    _C().gemm_fp8(a8, b8, view, sa, sb, True, variant)
    outside = torch.ones_like(buf, dtype=torch.bool)
    outside[16:16 + M, 32:32 + N] = False
    assert torch.equal(buf[outside], before[outside]), "the GEMM wrote outside its output view"
    want = before[16:16 + M, 32:32 + N].float() + _dequant_product(a8, sa, b8, sb)
    err = _worst_tile(view, want)
    print(f"\naccumulate {case} variant {variant}: worst-tile rel err {err:.3e}")
    assert err <= 1e-2, err
    # overwrite mode into the same view
    _C().gemm_fp8(a8, b8, view, sa, sb, False, variant)
    assert torch.equal(buf[outside], before[outside])
    assert _worst_tile(view, _dequant_product(a8, sa, b8, sb)) <= 1e-2


def test_gemm_fp8_rejects_unaligned_leading_dimensions():
    a8, sa, b8, sb = _operands(256, 512, 256, E4M3)
    out = torch.empty(256, 520, dtype=torch.bfloat16, device="cuda")[:, :512]   # ldc 520: not a multiple of 16
    with pytest.raises(RuntimeError, match="multiples of 16"):
        _C().gemm_fp8(a8, b8, out, sa, sb, False, 0)
    with pytest.raises(RuntimeError, match="float8_e4m3fn"):
        _C().gemm_fp8(b8, a8.to(torch.float32).to(E5M2), torch.empty(512, 256, dtype=torch.bfloat16, device="cuda"),
                      sb, sa, False, 0)


def test_gemm_fp8_nonfinite_scale_propagates():
    """An Inf in the input makes its scale 0 and its scale_inv Inf: the product must not come out finite."""
    x = _input((256, 512), "inf", seed=6)
    x8, _, sx = ops.fp8_cast(x, E4M3, transposed=False)
    w8, _, sw = ops.fp8_cast(_input((256, 512), "normal", seed=7), E4M3, transposed=False)
    y = ops.gemm_fp8(x8, sx, w8, sw)
    assert not bool(torch.isfinite(y).all())


# ------------------------------------------------------------------------------------------------------------------
# the fp8 training step
# ------------------------------------------------------------------------------------------------------------------
FP8_STEP_CASES = ["gqa-b2-s256-tied", "h2048-b1-s2048"]


@contextlib.contextmanager
def _fp8_engine(monkeypatch, case, lr=LR, **kw):
    from distributed_training_guide_b200.engine import TrainEngine

    base = engine_mod.get_config
    with monkeypatch.context() as mp:
        mp.setattr(engine_mod, "get_config", lambda name, **k: base(name, **{**case["overrides"], **k}))
        eng = TrainEngine.create(case["model"], parallelism="single", batch_size=case["B"], seq_length=case["S"],
                                 lr=lr, device="cuda", fp8=True, **kw)
    try:
        yield eng
    finally:
        eng.close()
        del eng
        gc.collect()
        torch.cuda.empty_cache()


def _torch_fp8_gemm(a8, scale_inv_a, b8, scale_inv_b, out=None, accumulate=False, out_dtype=torch.bfloat16):
    """PyTorch's fp8 GEMM (cuBLASLt through ``torch._scaled_mm``) on the same operands and scales."""
    r = torch._scaled_mm(a8, b8.t(), scale_a=scale_inv_a, scale_b=scale_inv_b, out_dtype=torch.float32,
                         use_fast_accum=False)
    if out is None:
        return r.to(out_dtype)
    out.copy_((out.float() + r) if accumulate else r)
    return out


def _torch_fp8_model_grads(config, weights, batches, monkeypatch):
    """Losses and gradients of a plain bf16 model whose decoder-layer projections use the same fp8 recipe with
    PyTorch's own ops: the reference casts and ``torch._scaled_mm``; every other op is PyTorch's bf16 op."""
    model = build_llama(config, dtype=torch.bfloat16, device="cuda", init=False)
    with torch.no_grad():
        for n, p in model.named_parameters():
            p.copy_(weights[n])
    model.fp8 = True
    losses = []
    with monkeypatch.context() as mp:
        mp.setattr(_ext, "_forced", {"all"})
        mp.setattr(ops, "gemm_fp8", _torch_fp8_gemm)
        for b in batches:
            out = model(input_ids=b["input_ids"].cuda(), labels=b["labels"].cuda())
            (out.loss / len(batches)).backward()
            losses.append(out.loss.item())
    grads = {n: p.grad.float() for n, p in model.named_parameters()}
    del model
    return losses, grads


# Gradients may be this much further from fp32 than the PyTorch-fp8 model's (factor; slack as the bf16 step test).
# Measured worst ratios: 1.18 (tied), 1.26 (H2048, layer 1 v_proj at step 3), 1.04 (accumulation).  Every gradient,
# those of the parameters that stay bf16 included, is 4e-2 to 2.5e-1 from fp32 in both fp8 models, against 5e-3 to
# 2e-2 for a bf16 step: the quantisation error of the projections reaches the embedding, norm and lm_head gradients
# through the activations, so those parameters are judged against the same fp8 yardstick, with the bf16 test's bound.
FP8_GRAD_FACTOR = 1.5


def _check_fp8_grads(tag, grads, ref_grads, fp8_grads, bf16_grads, report, failures):
    worst = 0.0
    for n, want in ref_grads.items():
        rk, r8, rb = _rel(grads[n], want), _rel(fp8_grads[n], want), _rel(bf16_grads[n], want)
        report.append((tag, n, rk, r8, rb))
        worst = max(worst, rk / max(r8, 1e-12))
        if rk > FP8_GRAD_FACTOR * r8 + GRAD_SLACK:
            failures.append(f"{tag} {n}: rel {rk:.3e} vs PyTorch fp8 {r8:.3e}")
    return worst


def _print_fp8_report(title, report):
    print(f"\n{title}\n{'':5}{'parameter':48} {'rel_kernel':>11} {'rel_torch8':>11} {'ratio':>7} {'rel_bf16':>11}")
    for tag, n, rk, r8, rb in report:
        print(f"{tag:5}{n:48} {rk:11.3e} {r8:11.3e} {rk / max(r8, 1e-12):7.2f} {rb:11.3e}")


@pytest.mark.parametrize("case", FP8_STEP_CASES)
def test_fp8_step_matches_fp32_reference(case, monkeypatch):
    cfg = CONFIGS[case]
    report, worst, failures = [], 0.0, []
    with _fp8_engine(monkeypatch, cfg) as eng:
        assert eng.model.fp8 and all(layer.fp8 for layer in eng.model.model.layers)
        rec = _capture_buckets(eng)
        config = eng.config
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
            (loss_fp8,), fp8_grads = _torch_fp8_model_grads(config, weights, [batch], monkeypatch)
            _, bf16_grads = _plain_model_grads(config, weights, [batch], torch.bfloat16, monkeypatch)
            print(f"\n{case} step {step}: loss kernel {loss:.5f} fp32 {loss_ref:.5f} torch-fp8 {loss_fp8:.5f}")
            if abs(loss - loss_ref) > LOSS_FACTOR * abs(loss_fp8 - loss_ref) + LOSS_SLACK:
                failures.append(f"step {step} loss {loss} fp32 {loss_ref} torch-fp8 {loss_fp8}")
            worst = max(worst, _check_fp8_grads(f"s{step}", _engine_grads(eng, rec), ref_grads, fp8_grads,
                                                bf16_grads, report, failures))
            _check_update(eng, rec, pre, step, lr)
            del ref_grads, fp8_grads, bf16_grads
    _print_fp8_report(f"{case} fp8: per-parameter gradient error vs fp32 (worst ratio to PyTorch fp8 {worst:.2f})",
                      report)
    assert not failures, "\n".join(failures)


def test_fp8_gradient_accumulation(monkeypatch):
    cfg, accum = CONFIGS["gqa-b2-s256"], 2
    report, failures = [], []
    with _fp8_engine(monkeypatch, cfg) as eng:
        rec = _capture_buckets(eng)
        model, strategy, config = eng.model, eng.strategy, eng.config
        batches = [eng.synthetic_batch(seed=20 + k) for k in range(accum)]
        weights = {n: p.detach().clone() for n, p in model.named_parameters()}
        pre = _pre_step_state(eng)
        lr = eng.optimizer.lr
        for k, b in enumerate(batches):
            out = model(**{n: t.cuda() for n, t in b.items()})
            with strategy.grad_sync(model, enabled=k == accum - 1):
                strategy.backward(model, out.loss / accum)
        eng.optimizer.step()
        eng.lr_scheduler.step()
        eng.optimizer.zero_grad(set_to_none=True)
        torch.cuda.synchronize()
        _check_order(eng, rec, "accumulation")
        _, ref_grads = _plain_model_grads(config, {n: w.float() for n, w in weights.items()}, batches, torch.float32,
                                          monkeypatch)
        _, fp8_grads = _torch_fp8_model_grads(config, weights, batches, monkeypatch)
        _, bf16_grads = _plain_model_grads(config, weights, batches, torch.bfloat16, monkeypatch)
        _check_fp8_grads("acc", _engine_grads(eng, rec), ref_grads, fp8_grads, bf16_grads, report, failures)
        _check_update(eng, rec, pre, 1, lr)
    _print_fp8_report("fp8 gradient accumulation (2 micro-batches): per-parameter gradient error", report)
    assert not failures, "\n".join(failures)


@pytest.mark.parametrize("case", ["gqa-b2-s256", "gqa-b2-s256-tied"])
def test_every_projection_runs_in_fp8(case, monkeypatch):
    """Per step: 12 x L fp8 GEMM launches (fwd, dgrad, wgrad of 4 projections in L layers) and only the lm_head's
    three bf16 GEMMs."""
    cfg = CONFIGS[case]
    counts = {"fp8": 0, "bf16": 0, "fp8_kernel": 0}
    real_fp8, real_bf16 = ops.gemm_fp8, ops.gemm

    def fp8(*a, **k):
        counts["fp8"] += 1
        return real_fp8(*a, **k)

    def bf16(*a, **k):
        counts["bf16"] += 1
        return real_bf16(*a, **k)

    with _fp8_engine(monkeypatch, cfg) as eng:
        L = eng.config.num_hidden_layers
        eng.step(eng.synthetic_batch(seed=0))   # warm-up outside the count
        with monkeypatch.context() as mp:
            mp.setattr(ops, "gemm_fp8", fp8)
            mp.setattr(ops, "gemm", bf16)
            n0 = _ext.launch_count()
            eng.step(eng.synthetic_batch(seed=1))
            torch.cuda.synchronize()
            launches = _ext.launch_count() - n0
    assert counts["fp8"] == 12 * L, counts
    assert counts["bf16"] == 3, counts
    print(f"\n{case}: {counts['fp8']} fp8 GEMMs, {counts['bf16']} bf16 GEMMs, {launches} own kernel launches per step")


# ------------------------------------------------------------------------------------------------------------------
# convergence
# ------------------------------------------------------------------------------------------------------------------
# measured on an H100: at most 4.0 % apart after step 10, both curves from 7.07 to below 0.3
CONV_STEPS, CONV_REL, CONV_LR = 100, 0.06, 2e-4


def _learnable_batches(vocab, B, S, steps, seed=0):
    """Shifted copies of one random sequence: the next token is a function of the current one."""
    g = torch.Generator().manual_seed(seed)
    base = torch.randint(0, vocab, (S + 64,), generator=g)
    out = []
    for i in range(steps):
        ids = torch.stack([base[(i * B + b) % 64:(i * B + b) % 64 + S] for b in range(B)])
        out.append({"input_ids": ids, "labels": ids.clone()})
    return out


def test_fp8_converges_like_bf16():
    from distributed_training_guide_b200.engine import TrainEngine

    curves = {}
    for fp8 in (False, True):
        eng = TrainEngine.create("debug-llama-gqa", parallelism="single", batch_size=2, seq_length=256, lr=CONV_LR,
                                 device="cuda", seed=0, fp8=fp8)
        batches = _learnable_batches(eng.config.vocab_size, 2, 256, CONV_STEPS)
        losses = [eng.step(b) for b in batches]
        curves[fp8] = [float(l) for l in losses]
        eng.close()
        del eng
        gc.collect()
        torch.cuda.empty_cache()
    bf16, fp8 = curves[False], curves[True]
    rel = [abs(f - b) / b for f, b in zip(fp8[10:], bf16[10:])]
    print("\nstep  bf16     fp8")
    for i in list(range(0, CONV_STEPS, 10)) + [CONV_STEPS - 1]:
        print(f"{i:4d}  {bf16[i]:.4f}  {fp8[i]:.4f}")
    print(f"max |fp8 - bf16| / bf16 after step 10: {max(rel):.4f}")
    v = math.log(1024)
    for c in (bf16, fp8):
        assert abs(c[0] - v) < 0.5, c[0]
        assert c[-1] < 1.0, c[-1]
    assert max(rel) <= CONV_REL, max(rel)


# ------------------------------------------------------------------------------------------------------------------
# multi-GPU
# ------------------------------------------------------------------------------------------------------------------
def _ddp_fp8_train(rank, world, steps):
    from distributed_training_guide_b200.engine import TrainEngine

    torch.manual_seed(0)
    eng = TrainEngine.create("debug-llama-gqa", parallelism="ddp", batch_size=2, seq_length=256, lr=1e-3, fp8=True)
    assert eng.model.fp8
    losses = [float(eng.step(eng.synthetic_batch(seed=i))) for i in range(steps)]
    sd = {k: v.detach().float().cpu() for k, v in eng.model.state_dict().items()}
    eng.close()
    return losses, sd


@pytest.mark.multigpu
def test_fp8_ddp_matches_single_gpu():
    from dist_utils import run_distributed
    from distributed_training_guide_b200.engine import TrainEngine

    world, steps = 2, 3
    res = run_distributed(_ddp_fp8_train, world=world, args=(steps,), timeout=300)
    torch.manual_seed(0)
    eng = TrainEngine.create("debug-llama-gqa", parallelism="single", batch_size=2, seq_length=256, lr=1e-3,
                             device="cuda", fp8=True)
    want = []
    for i in range(steps):
        parts = []
        for r in range(world):
            g = torch.Generator().manual_seed(1000 * i + r)
            parts.append(torch.randint(0, eng.config.vocab_size, (2, 256), generator=g))
        ids = torch.cat(parts)
        want.append(float(eng.step({"input_ids": ids, "labels": ids.clone()})))
    eng.close()
    import numpy as np

    (l0, sd0), (l1, sd1) = res
    for k in sd0:
        assert np.array_equal(sd0[k], sd1[k]), f"replicas diverged: {k}"
    for i in range(steps):
        assert abs(0.5 * (l0[i] + l1[i]) - want[i]) < 5e-2, (i, l0[i], l1[i], want[i])
