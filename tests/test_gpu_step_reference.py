"""The single-GPU training step against an fp32 reference model, parameter by parameter and step by step.

Every kernel has its own test against an fp32 op; this file checks that, put together, they compute the right
training step.  That step has machinery no single-kernel test reaches: gradients written straight into flat
buffers that are never zeroed (``zero_grad`` only resets counters, so each gradient must be overwritten on its
first use in a step and accumulated on later ones), fused q|k|v and gate|up weights over adjacent flat views, a
tied embedding written by two kernels, ops that work in place on autograd tensors (RoPE, the loss), and AdamW run
per bucket on a side stream inside backward (``DataParallelEngine`` with one rank, ``rs_adamw_kernel<1, ...>``).

Gradients: the engine's gradient of each parameter (captured as the AdamW kernel consumed it) against the fp32
gradient of the same weights and batch, judged relative to the error PyTorch's own bf16 ops make on the same
model (the bf16 noise floor).  Update: the engine's new parameters and moments against ``ref.adamw_step`` applied
to exactly what the kernel read, within one bf16 ulp per element.
"""
import contextlib
import gc
import math

import pytest
import torch

from distributed_training_guide_b200 import _ext
from distributed_training_guide_b200 import engine as engine_mod
from distributed_training_guide_b200.models.llama import build_llama
from distributed_training_guide_b200.ops import reference as ref

pytestmark = pytest.mark.gpu

# A correct bf16 step may be this much further from fp32 than PyTorch's bf16 ops are (factor, slack), and never
# further than the ceiling.
GRAD_FACTOR, GRAD_SLACK, GRAD_CEILING = 2.0, 5e-3, 3e-2
LOSS_FACTOR, LOSS_SLACK = 2.0, 2e-3
LR = 5e-3  # large enough that one AdamW step moves bf16 weights of magnitude 1 (the norm gains) by a whole ulp

CONFIGS = {
    "gqa-b2-s256": dict(model="debug-llama-gqa", B=2, S=256, overrides={}),
    "gqa-b2-s256-tied": dict(model="debug-llama-gqa", B=2, S=256, overrides=dict(tie_word_embeddings=True)),
    "gqa-b4-s128": dict(model="debug-llama-gqa", B=4, S=128, overrides={}),
    # GEMMs with several tiles per CTA on the 2-CTA variant; 16 q heads over 4 kv heads; V 32000
    "h2048-b1-s2048": dict(model="debug-llama-gqa", B=1, S=2048,
                           overrides=dict(hidden_size=2048, intermediate_size=5632, num_attention_heads=16,
                                          num_key_value_heads=4, vocab_size=32000, num_hidden_layers=2)),
}


# ------------------------------------------------------------------------------------------------------------------
# helpers
# ------------------------------------------------------------------------------------------------------------------
@contextlib.contextmanager
def _engine(monkeypatch, case, lr=LR):
    from distributed_training_guide_b200.engine import TrainEngine

    base = engine_mod.get_config
    with monkeypatch.context() as mp:
        mp.setattr(engine_mod, "get_config", lambda name, **kw: base(name, **{**case["overrides"], **kw}))
        eng = TrainEngine.create(case["model"], parallelism="single", batch_size=case["B"], seq_length=case["S"],
                                 lr=lr, device="cuda")
    try:
        yield eng
    finally:
        eng.close()
        del eng
        gc.collect()                # engines hold reference cycles: free their buffers before the next case
        torch.cuda.empty_cache()


def _capture_buckets(eng):
    """Record, for every bucket the engine launches, the gradient and parameters its AdamW kernel reads (cloned on
    the communication stream right before the kernel) and the launch order."""
    de = eng.strategy.engine
    rec = {"order": [], "grad": {}, "param": {}}
    run = de._run_bucket

    def capture(g, gbuf):
        rec["order"].append(g.name)
        rec["grad"][g.name] = g.grad.clone()
        rec["param"][g.name] = g.param.clone()
        return run(g, gbuf)

    de._run_bucket = capture
    return rec


@contextlib.contextmanager
def _fp32_matmuls():
    prev = torch.get_float32_matmul_precision()
    torch.set_float32_matmul_precision("highest")
    try:
        yield
    finally:
        torch.set_float32_matmul_precision(prev)


def _plain_model_grads(config, weights, batches, dtype, monkeypatch):
    """Losses and per-parameter gradients of a plain model (no flat groups, no engine) holding ``weights`` in
    ``dtype``, summed over ``batches`` with each loss divided by their number.  fp32: every op takes the
    ``ops/reference.py`` path (the op layer only sends bf16 to the kernels) with true fp32 matmuls.  bf16: every
    op is forced onto PyTorch's own bf16 ops (cuBLAS, flash SDPA)."""
    model = build_llama(config, dtype=dtype, device="cuda", init=False)
    with torch.no_grad():
        for n, p in model.named_parameters():
            p.copy_(weights[n])
    losses = []
    with monkeypatch.context() as mp, _fp32_matmuls():
        if dtype == torch.bfloat16:
            mp.setattr(_ext, "_forced", {"all"})
        for b in batches:
            out = model(input_ids=b["input_ids"].cuda(), labels=b["labels"].cuda())
            (out.loss / len(batches)).backward()
            losses.append(out.loss.item())
    grads = {n: p.grad.float() for n, p in model.named_parameters()}
    del model
    return losses, grads


def _engine_grads(eng, rec):
    """Per-parameter views of the flat gradients the AdamW kernels consumed."""
    out = {}
    for g in eng.strategy.groups:
        flat = rec["grad"][g.name]
        for n, o, shape in zip(g.names, g.offsets, g.shapes):
            out[n] = flat[o:o + math.prod(shape)].view(shape).float()
    return out


def _rel(a, b):
    return ((a - b).norm() / b.norm().clamp_min(1e-30)).item()


def _check_grads(tag, grads, ref_grads, bf16_grads, report):
    worst = 0.0
    for n, want in ref_grads.items():
        rk, rb = _rel(grads[n], want), _rel(bf16_grads[n], want)
        report.append((tag, n, rk, rb))
        worst = max(worst, rk / max(rb, 1e-12))
        assert rk <= GRAD_FACTOR * rb + GRAD_SLACK, f"{tag} {n}: rel {rk:.3e} vs bf16 floor {rb:.3e}"
        assert rk <= GRAD_CEILING, f"{tag} {n}: rel {rk:.3e} above the ceiling {GRAD_CEILING}"
    return worst


def _f32(x):
    """The value a kernel taking ``float`` receives for the Python float ``x``."""
    return float(torch.tensor(x, dtype=torch.float32))


def _bf16_spacing(x):
    """Distance between adjacent bf16 numbers at the magnitude of each element of ``x``."""
    _, e = torch.frexp(x.float().abs().clamp_min(torch.finfo(torch.bfloat16).tiny))
    return torch.ldexp(torch.ones_like(x, dtype=torch.float32), e - 8)


def _check_ulp(tag, got, want, operands=None):
    """Every element within one bf16 ulp.  The ulp is taken at the magnitude of the result or of ``operands``, the
    size of the terms the last addition of the update summed, whichever is larger: where ``p - step`` or
    ``b1 * m + (1 - b1) * g`` cancels, two correct fp32 evaluations differ by many ulps of the tiny result but by
    far less than one ulp of the terms.  Returns how many elements differ at all."""
    got_f, want_f = got.float(), want.float()
    mag = want_f.abs() if operands is None else torch.maximum(want_f.abs(), operands)
    ulps = (got_f - want_f).abs() / _bf16_spacing(mag)
    assert bool((ulps <= 1).all()), f"{tag}: {int((ulps > 1).sum())} elements more than 1 bf16 ulp off " \
                                    f"(worst {ulps.max().item():.3g})"
    return int((got != want).sum())


def _check_update(eng, rec, pre, step, lr):
    """The engine's new parameters and moments of every bucket against ``ref.adamw_step`` on bf16 copies of what
    the kernel read.  ``step`` and ``lr`` are what the step should have used, not what the engine passed."""
    opt = eng.optimizer
    b1, b2 = (_f32(b) for b in opt.param_groups[0]["betas"])
    eps, wd = _f32(opt.param_groups[0]["eps"]), _f32(opt.param_groups[0]["weight_decay"])
    ones, changed, total = 0, 0, 0
    for g in eng.strategy.groups:
        p0, m0, v0 = pre[g.name]
        assert torch.equal(rec["param"][g.name], p0), f"{g.name}: the AdamW kernel did not read the pre-step weights"
        st = opt.state[g.param]
        assert st["step"] == step, (g.name, st["step"], step)
        p, m, v, grad = p0.clone(), m0.clone(), v0.clone(), rec["grad"][g.name]
        ref.adamw_step(p, grad, m, v, _f32(lr), b1, b2, eps, wd, step, grad_scale=1.0)
        ones += _check_ulp(f"step {step} {g.name} exp_avg", st["exp_avg"], m,
                           b1 * m0.float().abs() + (1 - b1) * grad.float().abs())
        ones += _check_ulp(f"step {step} {g.name} exp_avg_sq", st["exp_avg_sq"], v)
        ones += _check_ulp(f"step {step} {g.name} params", g.param, p, p0.float().abs())
        changed += int((g.param != p0).sum())
        total += g.param.numel()
    assert changed > total // 2, f"step {step}: only {changed} of {total} weights changed: the check is vacuous"
    return ones


def _pre_step_state(eng):
    opt = eng.optimizer
    return {g.name: (g.param.clone(), opt.state[g.param]["exp_avg"].clone(), opt.state[g.param]["exp_avg_sq"].clone())
            for g in eng.strategy.groups}


def _check_order(eng, rec, tag):
    names = [g.name for g in eng.strategy.groups]
    assert sorted(rec["order"]) == sorted(names), f"{tag}: buckets launched {rec['order']}, expected each of {names} once"
    assert rec["order"][-1] == "embed", f"{tag}: the embedding bucket must be launched last: {rec['order']}"


def _print_report(title, report):
    print(f"\n{title}\n{'':4}{'parameter':48} {'rel_kernel':>11} {'rel_bf16':>11} {'ratio':>7}")
    for tag, n, rk, rb in report:
        print(f"{tag:4}{n:48} {rk:11.3e} {rb:11.3e} {rk / max(rb, 1e-12):7.2f}")


# ------------------------------------------------------------------------------------------------------------------
# A: three steps, each on its own batch
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", list(CONFIGS))
def test_step_matches_fp32_reference(case, monkeypatch):
    """Steps 2 and 3 are the point: a gradient that is accumulated where it should be overwritten, or left from
    the previous step, only shows once a step has run before."""
    cfg = CONFIGS[case]
    report, ulp_ones, worst = [], 0, 0.0
    with _engine(monkeypatch, cfg) as eng:
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
            (loss_bf16,), bf16_grads = _plain_model_grads(config, weights, [batch], torch.bfloat16, monkeypatch)
            assert abs(loss - loss_ref) <= LOSS_FACTOR * abs(loss_bf16 - loss_ref) + LOSS_SLACK, \
                (step, loss, loss_ref, loss_bf16)

            grads = _engine_grads(eng, rec)
            worst = max(worst, _check_grads(f"s{step}", grads, ref_grads, bf16_grads, report))
            if not config.tie_word_embeddings:
                # rows of tokens absent from this batch: exactly zero, not the previous step's gradient
                present = torch.zeros(config.vocab_size, dtype=torch.bool, device="cuda")
                present[batch["input_ids"].reshape(-1).cuda()] = True
                stale = grads["model.embed_tokens.weight"][~present]
                assert int(present.sum()) < config.vocab_size and int(torch.count_nonzero(stale)) == 0, \
                    f"step {step}: {int(torch.count_nonzero(stale.abs().sum(1)))} absent embedding rows are nonzero"
            ulp_ones += _check_update(eng, rec, pre, step, lr)
            del ref_grads, bf16_grads, grads
    _print_report(f"{case}: per-parameter gradient error (worst ratio {worst:.2f}; update elements one ulp off: "
                  f"{ulp_ones})", report)


# ------------------------------------------------------------------------------------------------------------------
# B: gradient accumulation, as trainer.py runs it
# ------------------------------------------------------------------------------------------------------------------
def test_gradient_accumulation_matches_reference(monkeypatch):
    """Two micro-batches per step (the first under ``grad_sync(enabled=False)``), two windows: GEMM accumulate into
    flat views, norm-gain and embedding accumulation, fused-weight counter resets, the loss's non-unit upstream
    gradient."""
    cfg, accum = CONFIGS["gqa-b2-s256"], 2
    report = []
    with _engine(monkeypatch, cfg) as eng:
        rec = _capture_buckets(eng)
        model, strategy, config = eng.model, eng.strategy, eng.config
        for window in (1, 2):
            batches = [eng.synthetic_batch(seed=10 * window + k) for k in range(accum)]
            weights = {n: p.detach().clone() for n, p in model.named_parameters()}
            pre = _pre_step_state(eng)
            lr = eng.optimizer.lr
            rec["order"].clear()
            for k, b in enumerate(batches):
                out = model(**{n: t.cuda() for n, t in b.items()})
                with strategy.grad_sync(model, enabled=k == accum - 1):
                    strategy.backward(model, out.loss / accum)
                if k < accum - 1:
                    torch.cuda.synchronize()
                    assert not rec["order"], f"window {window}: buckets launched inside the accumulation window"
            eng.optimizer.step()
            eng.lr_scheduler.step()
            eng.optimizer.zero_grad(set_to_none=True)
            torch.cuda.synchronize()
            _check_order(eng, rec, f"window {window}")
            _, ref_grads = _plain_model_grads(config, {n: w.float() for n, w in weights.items()}, batches,
                                              torch.float32, monkeypatch)
            _, bf16_grads = _plain_model_grads(config, weights, batches, torch.bfloat16, monkeypatch)
            _check_grads(f"w{window}", _engine_grads(eng, rec), ref_grads, bf16_grads, report)
            _check_update(eng, rec, pre, window, lr)
    _print_report("gradient accumulation: per-parameter gradient error", report)


# ------------------------------------------------------------------------------------------------------------------
# C: the optimizer kernels of the single-GPU step
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kernel", ["rs_adamw", "adamw_flat"])
@pytest.mark.parametrize("state_dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("grad_scale", [1.0, 0.5])
@pytest.mark.parametrize("first_step", [1, 1000])
def test_bucket_adamw_single_rank(kernel, state_dtype, grad_scale, first_step):
    """``rs_adamw_kernel<1, ...>`` (what ``SingleDevice`` runs for every bucket, through ``SymmGroup(ranks=[0])``)
    and ``adamw_flat``: five consecutive steps with fresh gradients, moments carried from step to step, against
    ``ref.adamw_step`` on the same storage dtypes.  Each step is checked on what the kernel read, so one step's
    rounding does not compound into the next.  A run starting at step 1000 has bias corrections close to 1."""
    from distributed_training_guide_b200.parallel.symm import SymmGroup

    n, lr, b1, b2, eps, wd = 8 * 123457, 1e-2, 0.9, 0.999, 1e-8, 0.1
    f = (_f32(lr), _f32(b1), _f32(b2), _f32(eps), _f32(wd))
    dev = torch.device("cuda", 0)
    gen = torch.Generator(device=dev).manual_seed(first_step)
    sg = SymmGroup(dev, ranks=[0])
    try:
        gbuf, pbuf = sg.alloc(n, torch.bfloat16), sg.alloc(n, torch.bfloat16)
        p, g = pbuf.local, gbuf.local
        p.copy_(0.05 * torch.randn(n, device=dev, generator=gen))
        if first_step == 1:
            m = torch.zeros(n, device=dev, dtype=state_dtype)
            v = torch.zeros(n, device=dev, dtype=state_dtype)
        else:   # a run in progress: moments of the size the gradients below give
            m = (1e-3 * torch.randn(n, device=dev, generator=gen)).to(state_dtype)
            v = (1e-2 * torch.randn(n, device=dev, generator=gen)).square().to(state_dtype)
        ones, changed = 0, 0
        for step in range(first_step, first_step + 5):
            g.copy_(1e-2 * torch.randn(n, device=dev, generator=gen))
            p0, m0, v0 = p.clone(), m.clone(), v.clone()
            if kernel == "rs_adamw":
                sg.rs_adamw_(gbuf, pbuf, None, m, v, True, 0, n, (lr, b1, b2, eps, wd), step, grad_scale)
            else:
                _ext.load(True).adamw_flat(p, g, m, v, lr, b1, b2, eps, wd, step, grad_scale)
            torch.cuda.synchronize()
            pr, mr, vr = p0.clone(), m0.clone(), v0.clone()
            ref.adamw_step(pr, g, mr, vr, *f, step, grad_scale=grad_scale)
            m_scale = b1 * m0.float().abs() + (1 - b1) * (g.float() * grad_scale).abs()
            if state_dtype == torch.bfloat16:
                ones += _check_ulp(f"step {step} exp_avg", m, mr, m_scale)
                ones += _check_ulp(f"step {step} exp_avg_sq", v, vr)
            else:
                # 1e-6 of the operands: b1*m + (1-b1)*g can cancel, and the kernel may fuse it into one FMA
                assert ((m - mr).abs() <= 1e-6 * m_scale).all(), \
                    f"step {step} exp_avg: max rel {((m - mr).abs() / m_scale.clamp_min(1e-30)).max().item():.3g}"
                assert ((v - vr).abs() <= 1e-6 * vr.abs()).all(), \
                    f"step {step} exp_avg_sq: max rel {((v - vr).abs() / vr.abs().clamp_min(1e-30)).max().item():.3g}"
            ones += _check_ulp(f"step {step} params", p, pr, p0.float().abs())
            changed += int((p != p0).sum())
        sg.check()
        assert changed > 5 * n // 2, f"only {changed} of {5 * n} parameter updates moved a bf16 weight"
        print(f"\n{kernel} state {state_dtype} grad_scale {grad_scale} from step {first_step}: "
              f"{ones} elements differ (by at most one ulp) over 5 steps")
    finally:
        sg.close()
