"""Gradient clipping on the GPU (``csrc/grad_clip.cu`` through ``DataParallelEngine``): the reduce + sum-of-squares
kernel against an fp64 norm, the clipped single-GPU step against ``ref.adamw_step`` with the same coefficient, the
flag at a huge ``max_norm`` against the engine without it, and (>= 2 GPUs) the ZeRO-1 and all-reduce engines with
the peer-pointer and the NVLS kernels."""
import contextlib
import gc
import math

import numpy as np
import pytest
import torch

from dist_utils import run_distributed

pytestmark = pytest.mark.gpu

CASES = {
    "gqa-b2-s256": dict(B=2, S=256, overrides={}),
    "gqa-b2-s256-tied": dict(B=2, S=256, overrides=dict(tie_word_embeddings=True)),
    "gqa-b4-s128": dict(B=4, S=128, overrides={}),
}
LR = 5e-3


def _f32(x):
    return float(torch.tensor(x, dtype=torch.float32))


def _bf16_spacing(x):
    _, e = torch.frexp(x.float().abs().clamp_min(torch.finfo(torch.bfloat16).tiny))
    return torch.ldexp(torch.ones_like(x, dtype=torch.float32), e - 8)


def _check_ulp(tag, got, want, operands=None):
    """Every element within one bf16 ulp of the result or of the terms its last addition summed."""
    got_f, want_f = got.float(), want.float()
    mag = want_f.abs() if operands is None else torch.maximum(want_f.abs(), operands)
    ulps = (got_f - want_f).abs() / _bf16_spacing(mag)
    assert bool((ulps <= 1).all()), f"{tag}: {int((ulps > 1).sum())} elements more than 1 bf16 ulp off " \
                                    f"(worst {ulps.max().item():.3g})"


def _param_norm64(groups, flats):
    """fp64 L2 norm of the flat gradients ``flats[name]`` over each group's parameter elements."""
    total = 0.0
    for g in groups:
        for o, shape in zip(g.offsets, g.shapes):
            total += float(flats[g.name][o:o + math.prod(shape)].double().square().sum())
    return math.sqrt(total)


@contextlib.contextmanager
def _engine(monkeypatch, case, **kw):
    from distributed_training_guide_b200 import engine as engine_mod
    from distributed_training_guide_b200.engine import TrainEngine

    base = engine_mod.get_config
    with monkeypatch.context() as mp:
        mp.setattr(engine_mod, "get_config", lambda name, **k: base(name, **{**case["overrides"], **k}))
        torch.manual_seed(0)
        eng = TrainEngine.create("debug-llama-gqa", parallelism="single", batch_size=case["B"], seq_length=case["S"],
                                 lr=LR, device="cuda", **kw)
    try:
        yield eng
    finally:
        eng.close()
        del eng
        gc.collect()
        torch.cuda.empty_cache()


def _capture(eng, rel_max_norm=None):
    """Clone every bucket's gradient as the reduce kernel reads it (one rank: exactly what AdamW consumes).  With
    ``rel_max_norm``, set ``max_grad_norm`` to that fraction of the step's fp64 norm before the clipped update."""
    de = eng.strategy.engine
    rec = {"grad": {}}
    run, step = de._run_bucket, de._clipped_step

    def capture(g, gbuf):
        rec["grad"][g.name] = g.grad.clone()
        return run(g, gbuf)

    def clipped_step():
        torch.cuda.synchronize()
        rec["norm64"] = _param_norm64(eng.strategy.groups, rec["grad"])
        if rel_max_norm is not None:
            eng.optimizer.max_grad_norm = rel_max_norm * rec["norm64"]
        return step()

    de._run_bucket, de._clipped_step = capture, clipped_step
    return rec


# ------------------------------------------------------------------------------------------------------------------
# the norm kernel against fp64
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("sizes", [[5, 13, 24], [1000, 7, 4096 * 3 + 1], [3_000_001, 16, 1_048_576 + 3]],
                         ids=["tiny", "partial-vectors", "grid-stride"])
@pytest.mark.parametrize("scale", [1.0, 0.5])
def test_reduce_sumsq_against_fp64(sizes, scale):
    from distributed_training_guide_b200.ops import reference as ref
    from distributed_training_guide_b200.parallel.symm import SymmGroup

    dev = torch.device("cuda", 0)
    sg = SymmGroup(dev, ranks=[0])
    try:
        ranges, off = [], 0
        for n in sizes:                      # parameters at 8-element offsets, as in a flat group
            ranges.append([off, off + n])
            off = (off + n + 7) // 8 * 8
        n_total = (off + 255) // 256 * 256 + 256   # and a padded tail
        buf = sg.alloc(n_total, torch.bfloat16)
        gen = torch.Generator(device=dev).manual_seed(len(sizes) + sum(sizes))
        x = torch.full((n_total,), float("nan"), device=dev, dtype=torch.bfloat16)   # NaN padding
        for b, e in ranges:
            x[b:e] = (torch.randn(e - b, device=dev, generator=gen) * 3).to(torch.bfloat16)
        table = torch.tensor(ranges, dtype=torch.int64, device=dev)
        blocks = sg.comm_blocks
        partials = torch.zeros(2 * blocks, dtype=torch.float64, device=dev)
        slots = sg.alloc(2, torch.float64)
        outs = []
        for call in range(2):
            buf.local.copy_(x)
            partials.fill_(float("nan"))
            sg.reduce_sumsq_(buf, 0, n_total, scale, False, table, partials[:blocks])
            partials[blocks:] = 0
            out = torch.zeros(2, dtype=torch.float32, device=dev)
            sg.clip_finalize_(partials, slots, call, 1.0, 1.0, out)
            torch.cuda.synchronize()
            outs.append(out.clone())
        sg.check()
        stored = (x.float() * scale).to(torch.bfloat16)
        inside = torch.zeros(n_total, dtype=torch.bool, device=dev)
        for b, e in ranges:
            inside[b:e] = True
        assert torch.equal(buf.local[inside], stored[inside]), "the stored reduced gradient is not round(x * scale)"
        want = math.sqrt(float(stored[inside].double().square().sum()))
        norm, coef = float(outs[0][0]), outs[0][1]
        assert math.isfinite(norm), "padding reached the norm"
        assert abs(norm - want) <= 2e-6 * want, (norm, want)
        assert torch.equal(coef.cpu(), ref.clip_coefficient(outs[0][0].cpu(), 1.0)), (float(coef), norm)
        assert torch.equal(outs[0], outs[1]), "two calls gave different bits"
    finally:
        sg.close()


# ------------------------------------------------------------------------------------------------------------------
# the clipped single-GPU step
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", list(CASES))
def test_clipped_step_matches_reference_update(case, monkeypatch):
    from distributed_training_guide_b200.ops import reference as ref

    with _engine(monkeypatch, CASES[case], max_grad_norm=1.0) as eng:
        rec = _capture(eng, rel_max_norm=0.1)
        opt = eng.optimizer
        b1, b2 = (_f32(b) for b in opt.param_groups[0]["betas"])
        eps, wd = _f32(opt.param_groups[0]["eps"]), _f32(opt.param_groups[0]["weight_decay"])
        for step in (1, 2, 3):
            pre = {g.name: (g.param.clone(), opt.state[g.param]["exp_avg"].clone(),
                            opt.state[g.param]["exp_avg_sq"].clone()) for g in eng.strategy.groups}
            lr = opt.lr
            eng.step(eng.synthetic_batch(seed=step))
            torch.cuda.synchronize()
            norm = eng.grad_norm()
            coef = eng.strategy.engine._clip_out[1].clone()
            assert abs(float(norm) - rec["norm64"]) <= 2e-6 * rec["norm64"], (step, float(norm), rec["norm64"])
            assert torch.equal(coef.cpu(), ref.clip_coefficient(norm.cpu(), opt.max_grad_norm))
            assert 0.05 < float(coef) < 0.2, float(coef)
            for g in eng.strategy.groups:
                p0, m0, v0 = pre[g.name]
                p, m, v, grad = p0.clone(), m0.clone(), v0.clone(), rec["grad"][g.name]
                ref.adamw_step(p, grad, m, v, _f32(lr), b1, b2, eps, wd, step, grad_scale=1.0, coef=coef)
                st = opt.state[g.param]
                cg = grad.float() * coef
                _check_ulp(f"step {step} {g.name} exp_avg", st["exp_avg"], m,
                           b1 * m0.float().abs() + (1 - b1) * cg.abs())
                _check_ulp(f"step {step} {g.name} exp_avg_sq", st["exp_avg_sq"], v)
                _check_ulp(f"step {step} {g.name} params", g.param, p, p0.float().abs())


def test_huge_max_norm_is_bit_identical_to_no_clipping(monkeypatch):
    """One rank: the deferred path feeds AdamW the same bf16 gradient, and coef is exactly 1."""
    case = CASES["gqa-b2-s256"]
    states = []
    for kw in ({}, {"max_grad_norm": 1e30}):
        with _engine(monkeypatch, case, **kw) as eng:
            for step in range(3):
                eng.step(eng.synthetic_batch(seed=step))
            torch.cuda.synchronize()
            if kw:
                assert float(eng.strategy.engine._clip_out[1]) == 1.0
                assert math.isfinite(float(eng.grad_norm()))
            else:
                assert eng.grad_norm() is None
            opt = eng.optimizer
            states.append({g.name: (g.param.clone(), opt.state[g.param]["exp_avg"].clone(),
                                    opt.state[g.param]["exp_avg_sq"].clone()) for g in eng.strategy.groups})
    for name, (p, m, v) in states[0].items():
        p1, m1, v1 = states[1][name]
        assert torch.equal(p, p1) and torch.equal(m, m1) and torch.equal(v, v1), name


@pytest.mark.parametrize("feature", ["fp8", "document_masking"])
def test_clipping_combines_with(feature, monkeypatch):
    case = CASES["gqa-b2-s256"]
    with _engine(monkeypatch, case, max_grad_norm=1e-3, **{feature: True}) as eng:
        rec = _capture(eng)
        batch = eng.synthetic_batch(seed=0)
        if feature == "document_masking":
            pos = torch.cat([torch.arange(100), torch.arange(case["S"] - 100)])
            batch["position_ids"] = pos.expand(case["B"], -1).contiguous()
        loss = float(eng.step(batch))
        torch.cuda.synchronize()
        assert math.isfinite(loss)
        norm = float(eng.grad_norm())
        assert abs(norm - rec["norm64"]) <= 2e-6 * rec["norm64"], (norm, rec["norm64"])
        assert float(eng.strategy.engine._clip_out[1]) < 1.0


# ------------------------------------------------------------------------------------------------------------------
# >= 2 GPUs: ZeRO-1 and all-reduce, peer-pointer and NVLS kernels
# ------------------------------------------------------------------------------------------------------------------
MAX_NORM = 1e-3


def _dp_train(rank, world, parallelism, nvls, max_norm, steps):
    import os

    os.environ["DTG_NVLS"] = nvls
    import torch.distributed as dist

    from distributed_training_guide_b200.engine import TrainEngine

    torch.manual_seed(0)
    eng = TrainEngine.create("debug-llama-gqa", parallelism=parallelism, batch_size=2, seq_length=256, lr=1e-3,
                             max_grad_norm=max_norm)
    multicast = bool(eng.strategy.symm.nvls)
    rec = _capture(eng) if max_norm is not None else None
    norms, mean_norms = [], []
    for i in range(steps):
        eng.step(eng.synthetic_batch(seed=i))
        torch.cuda.synchronize()
        if max_norm is None:
            continue
        norms.append(float(eng.grad_norm()))
        # fp64 norm of the rank-mean gradient
        local = torch.cat([rec["grad"][g.name][o:o + math.prod(s)].double()
                           for g in eng.strategy.groups for o, s in zip(g.offsets, g.shapes)])
        dist.all_reduce(local)
        mean_norms.append(float((local / world).norm()))
    sd = {k: v.detach().float().cpu() for k, v in eng.model.state_dict().items()}
    eng.close()
    return norms, mean_norms, sd, multicast


def _single_run(steps, world, max_norm):
    from distributed_training_guide_b200.engine import TrainEngine

    torch.manual_seed(0)
    eng = TrainEngine.create("debug-llama-gqa", parallelism="single", batch_size=2 * world, seq_length=256, lr=1e-3,
                             device="cuda", max_grad_norm=max_norm)
    for i in range(steps):
        parts = [torch.randint(0, eng.config.vocab_size, (2, 256), generator=torch.Generator().manual_seed(1000 * i + r))
                 for r in range(world)]
        ids = torch.cat(parts)
        eng.step({"input_ids": ids, "labels": ids.clone()})
    sd = {k: v.detach().float().cpu().numpy() for k, v in eng.model.state_dict().items()}
    eng.close()
    return sd


@pytest.mark.multigpu
@pytest.mark.parametrize("nvls", ["1", "0"], ids=["nvls", "pull"])
@pytest.mark.parametrize("parallelism", ["ddp", "ddp_allreduce"])
def test_data_parallel_clipping(parallelism, nvls):
    world, steps = 2, 3
    res = run_distributed(_dp_train, world=world, args=(parallelism, nvls, MAX_NORM, steps), timeout=600)
    (n0, m0, sd0, mc), (n1, _, sd1, _) = res
    assert [np.float32(a).tobytes() for a in n0] == [np.float32(a).tobytes() for a in n1], (n0, n1)
    for k in sd0:
        assert np.array_equal(sd0[k], sd1[k]), f"replicas diverged: {k}"
    for got, want in zip(n0, m0):
        assert got > MAX_NORM
        assert abs(got - want) <= 4e-3 * want, (got, want)   # the stored mean is rounded to bf16 once
    ref = _single_run(steps, world, MAX_NORM)
    for k in sd0:
        assert np.abs(sd0[k] - ref[k]).max() < 5e-2, k
    if nvls == "1" and not mc:
        pytest.skip("no NVSwitch multicast on this system: the NVLS kernels were not exercised")


@pytest.mark.multigpu
@pytest.mark.parametrize("nvls", ["1", "0"], ids=["nvls", "pull"])
def test_data_parallel_huge_max_norm_matches_no_clipping(nvls):
    world, steps = 2, 3
    _, _, sd_on, mc = run_distributed(_dp_train, world=world, args=("ddp", nvls, 1e30, steps), timeout=600)[0]
    _, _, sd_off, _ = run_distributed(_dp_train, world=world, args=("ddp", nvls, None, steps), timeout=600)[0]
    if nvls == "1" and mc:
        # the in-switch reduction returns bf16 and 1/N is exact: AdamW reads the same gradient bits
        for k in sd_on:
            assert np.array_equal(sd_on[k], sd_off[k]), k
    else:
        # the pull path rounds the fp32 sum of the peers' gradients to bf16 once before AdamW; where a gradient is
        # near zero that can flip the sign of one lr-sized AdamW step (lr 1e-3, 3 steps), nowhere more
        diffs = {k: float(np.abs(sd_on[k] - sd_off[k]).max()) for k in sd_on}
        assert max(diffs.values()) <= 2 * 1e-3 * steps + 1e-2 * max(float(np.abs(v).max()) for v in sd_off.values()) \
            * 2 ** -8, diffs
        changed = sum(int((sd_on[k] != sd_off[k]).sum()) for k in sd_on)
        total = sum(v.size for v in sd_on.values())
        assert changed < total // 10, f"{changed} of {total} weights differ: more than rounding"
    if nvls == "1" and not mc:
        pytest.skip("no NVSwitch multicast on this system: the NVLS kernels were not exercised")
