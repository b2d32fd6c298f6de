"""OLMo 2 on one GPU.

Kernels, element by element against fp64:
  * full-width QK-norm + RoPE (``qk_norm_full_rope_fwd`` / ``_bwd``) at the head counts of debug-olmo2 (4:2), 7B
    (32:32), 13B (40:40) and 32B (40:8), with shared and per-token tables, zero and negative gains, an all-zero q
    region, magnitudes near the top of bf16's range and token counts that leave the backward's CTAs uneven.  Forward
    outputs may differ from the exact ``rope(rmsnorm(x) * w)`` by two bf16 roundings (``bf16(x * rstd * w)`` and the
    stored output) of the terms the rotation sums; ``dx`` by one bf16 rounding plus fp32 error on the terms of
    ``rstd * (g - xhat * mean(g * xhat))`` (the inverse rotation's terms included, since it may cancel); the gain
    gradients by fp32 error relative to the sum of their terms' magnitudes.  The backward is bit-identical run to run.
  * norm-then-add (``rmsnorm_add_fwd``): bit-identical to ``rmsnorm_fwd`` followed by a bf16 add at every hidden-size
    instantiation, within two bf16 roundings of fp64, and its backward (``ops.rms_norm_add``) against fp64 autograd.

Training: three single-GPU steps of debug-olmo2, untied and tied, against an fp32 reference model parameter by
parameter (the helpers of ``test_gpu_step_reference.py``); a packed-document step; chapter 01 plain and with --fp8,
with checkpoint and resume."""
import json
import math

import pytest
import torch

from distributed_training_guide_b200 import _ext, ops
from distributed_training_guide_b200.ops import reference as ref
from test_gpu_chapters import ROOT, _run
from test_gpu_qwen3 import _plain_grads_docmask, _positions_from_starts
from test_gpu_step_reference import (LOSS_FACTOR, LOSS_SLACK, _capture_buckets, _check_grads, _check_order,
                                     _check_update, _engine, _engine_grads, _plain_model_grads, _pre_step_state,
                                     _print_report)

pytestmark = pytest.mark.gpu

EPS = 1e-6
U = 2.0 ** -8   # bf16 unit roundoff


def _C():
    return _ext.load(required=True)


# ------------------------------------------------------------------------------------------------------------------
# full-width QK-norm + RoPE
# ------------------------------------------------------------------------------------------------------------------
def _rope64(x, cos, sin, inverse=False):
    c, s = cos.double(), sin.double()
    if c.dim() == 2:
        c, s = c[None, :, None, :], s[None, :, None, :]
    else:
        c, s = c[:, :, None, :], s[:, :, None, :]
    if inverse:
        s = -s
    x1, x2 = x[..., :64], x[..., 64:]
    return torch.cat([x1 * c - x2 * s, x2 * c + x1 * s], dim=-1), torch.cat(
        [x1.abs() * c.abs() + x2.abs() * s.abs(), x2.abs() * c.abs() + x1.abs() * s.abs()], dim=-1)


def _fp64(qkv, q_w, k_w, cos, sin, nh, nkv, dout):
    """Exact forward output, its magnitude terms, dx, dx's magnitude terms, dw [(nh+nkv)*128] and dw's term sums."""
    B, S = qkv.shape[:2]
    x = qkv[:, :, :nh + nkv].double()
    w = torch.cat([q_w.double(), k_w.double()]).view(nh + nkv, 128)

    def region_rstd(r):   # [B, S, n, 128] -> [B, S, 1, 1]
        return 1.0 / torch.sqrt(r.square().mean((-2, -1), keepdim=True) + EPS)

    rstd = torch.cat([region_rstd(x[:, :, :nh]).expand(B, S, nh, 1), region_rstd(x[:, :, nh:]).expand(B, S, nkv, 1)],
                     dim=2)
    xh = x * rstd
    out, mag = _rope64(xh * w, cos, sin)
    d, dmag = _rope64(dout[:, :, :nh + nkv].double(), cos, sin, inverse=True)
    g = d * w
    gx, agx = g * xh, (dmag * w * xh).abs()
    dot = torch.cat([gx[:, :, :nh].mean((-2, -1), keepdim=True).expand(B, S, nh, 1),
                     gx[:, :, nh:].mean((-2, -1), keepdim=True).expand(B, S, nkv, 1)], dim=2)
    adot = torch.cat([agx[:, :, :nh].mean((-2, -1), keepdim=True).expand(B, S, nh, 1),
                      agx[:, :, nh:].mean((-2, -1), keepdim=True).expand(B, S, nkv, 1)], dim=2)
    dx = rstd * (g - xh * dot)
    # fp32 error scales with the terms the kernel sums, the inverse rotation's included (it may cancel)
    dx_mag = rstd * ((dmag * w).abs() + xh.abs() * adot)
    dw = (d * xh).sum((0, 1)).reshape(-1)
    dw_mag = (dmag * xh).abs().sum((0, 1)).reshape(-1)
    return out, mag, dx, dx_mag, dw, dw_mag


def _case(B, S, nh, nkv, per_token, seed, scale=1.0, zero_region=False, gains="random"):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    qkv = (torch.randn(B, S, nh + 2 * nkv, 128, generator=gen, device="cuda") * scale).to(torch.bfloat16)
    if zero_region:   # one token's whole q region, another token's whole k region
        qkv[:, 1, :nh] = 0
        qkv[:, -1, nh:nh + nkv] = 0
    q_w = torch.randn(nh * 128, generator=gen, device="cuda").to(torch.bfloat16)
    k_w = torch.randn(nkv * 128, generator=gen, device="cuda").to(torch.bfloat16)
    if gains == "zeros-and-negatives":
        q_w[::5] = 0
        k_w[3::7] = 0
        k_w[:128] = 0   # a whole k head's gain
        q_w[1::3] = -q_w[1::3].abs()
        k_w[::2] = -k_w[::2].abs()
    pos = torch.randint(0, 4096, (B, S), generator=gen, device="cuda") if per_token else torch.arange(S, device="cuda")
    cos, sin = ref.rope_tables(pos, 128, 5e5)
    dout = torch.randn(B, S, nh + 2 * nkv, 128, generator=gen, device="cuda").to(torch.bfloat16)
    return qkv, q_w, k_w, cos, sin, dout


CASES = {
    # T = 3 * 77 = 231 tokens, fewer than the backward's CTAs
    "debug-4-2-ragged": dict(B=3, S=77, nh=4, nkv=2, per_token=False),
    "debug-4-2-one-token": dict(B=1, S=1, nh=4, nkv=2, per_token=True),
    "7b-32-32-per-token": dict(B=2, S=300, nh=32, nkv=32, per_token=True),
    "13b-40-40": dict(B=1, S=1000, nh=40, nkv=40, per_token=False),
    "13b-40-40-zero-negative-gains": dict(B=2, S=129, nh=40, nkv=40, per_token=True, gains="zeros-and-negatives"),
    "32b-40-8-zero-regions": dict(B=2, S=64, nh=40, nkv=8, per_token=False, zero_region=True),
    # |x| up to ~2^126: the sums of squares take the scaled path
    "32b-40-8-near-bf16-limit": dict(B=1, S=40, nh=40, nkv=8, per_token=False, scale=2e37),
    "7b-32-32-tiny": dict(B=1, S=40, nh=32, nkv=32, per_token=False, scale=1e-30),
    # T = 4095: more tokens than the backward's CTAs, split unevenly among them
    "7b-32-32-long-ragged": dict(B=1, S=4095, nh=32, nkv=32, per_token=False),
}


@pytest.mark.parametrize("case", list(CASES))
def test_full_width_kernels_against_fp64(case):
    c = dict(CASES[case])
    B, S, nh, nkv, per_token = c.pop("B"), c.pop("S"), c.pop("nh"), c.pop("nkv"), c.pop("per_token")
    qkv, q_w, k_w, cos, sin, dout = _case(B, S, nh, nkv, per_token, seed=len(case), **c)
    assert torch.isfinite(qkv.float()).all()
    if c.get("scale", 1.0) > 1e30:
        assert qkv.float().abs().max() >= 2.0 ** 56
    out64, mag, dx64, dx_mag, dw64, dw_mag = _fp64(qkv, q_w, k_w, cos, sin, nh, nkv, dout)
    C = _C()
    x = qkv.clone()
    x_save, rstd = C.qk_norm_full_rope_fwd(x, q_w, k_w, cos, sin, nh, nkv, EPS)
    torch.cuda.synchronize()
    assert x_save.shape == (B, S, nh + nkv, 128) and rstd.shape == (B, S, 2)
    assert torch.equal(x[:, :, nh + nkv:], qkv[:, :, nh + nkv:]), "V heads changed"
    assert torch.equal(x_save, qkv[:, :, :nh + nkv]), "the saved pre-norm heads differ from the input"
    got = x[:, :, :nh + nkv].double()
    assert torch.isfinite(got).all()
    err = (got - out64).abs()
    bound = 2 * U * (1 + 1e-5) * mag + 1e-38
    assert bool((err <= bound).all()), f"forward: {int((err > bound).sum())} elements off, worst " \
                                       f"{(err / bound).max().item():.3g} of the bound"
    if c.get("zero_region"):
        assert torch.equal(x[:, 1, :nh], torch.zeros_like(x[:, 1, :nh]))
        torch.testing.assert_close(rstd[:, 1, 0].double(), torch.full_like(rstd[:, 1, 0].double(), 1 / math.sqrt(EPS)),
                                   rtol=1e-6, atol=0)

    d = dout.clone()
    dw = C.qk_norm_full_rope_bwd(d, x_save, rstd, q_w, k_w, cos, sin, nh, nkv)
    torch.cuda.synchronize()
    assert dw.shape == ((nh + nkv) * 128,) and dw.dtype == torch.float32
    assert torch.equal(d[:, :, nh + nkv:], dout[:, :, nh + nkv:]), "dV changed"
    derr = (d[:, :, :nh + nkv].double() - dx64).abs()
    dbound = U * dx64.abs() + 1e-5 * dx_mag + 1e-38
    assert bool((derr <= dbound).all()), f"dx: {int((derr > dbound).sum())} elements off, worst " \
                                         f"{(derr / dbound).max().item():.3g} of the bound"
    werr = (dw.double() - dw64).abs()
    wbound = 1e-5 * dw_mag + 1e-38
    assert bool((werr <= wbound).all()), f"dw: worst {(werr / wbound).max().item():.3g} of the bound"
    # the same backward again: bit-identical (fixed-order reduction, no atomics)
    d2 = dout.clone()
    dw2 = C.qk_norm_full_rope_bwd(d2, x_save, rstd, q_w, k_w, cos, sin, nh, nkv)
    assert torch.equal(dw, dw2) and torch.equal(d, d2)


def test_op_matches_kernels_and_accumulates_in_flat_buffers():
    """``ops.olmo_qk_norm_rope_`` through autograd with the gains carrying flat-gradient views, as the engines run it:
    the first micro-batch overwrites stale gradient contents, the second accumulates."""
    B, S, nh, nkv = 2, 128, 8, 2
    nq, nk = nh * 128, nkv * 128
    q_w = torch.nn.Parameter(torch.randn(nq, device="cuda").to(torch.bfloat16))
    k_w = torch.nn.Parameter(torch.randn(nk, device="cuda").to(torch.bfloat16))
    flat = torch.full((nq + nk,), 123.0, device="cuda", dtype=torch.bfloat16)   # stale contents
    q_w._dtg_grad, k_w._dtg_grad = flat[:nq], flat[nq:]
    q_w._dtg_writes = k_w._dtg_writes = 0
    want = torch.zeros(nq + nk, dtype=torch.float64, device="cuda")
    tol = torch.zeros_like(want)
    for mb in range(2):
        qkv, _, _, cos, sin, dout = _case(B, S, nh, nkv, False, seed=10 + mb)
        out64, _, dx64, dx_mag, dw64, dw_mag = _fp64(qkv, q_w.detach(), k_w.detach(), cos, sin, nh, nkv, dout)
        want += dw64
        tol += U * dw64.abs() + 1e-5 * dw_mag   # one bf16 rounding per write of the running sum, fp32 noise
        leaf = qkv.clone().requires_grad_(True)
        out = ops.olmo_qk_norm_rope_(leaf * 1, q_w, k_w, cos, sin, nh, nkv, EPS)
        assert bool(((out[:, :, :nh + nkv].double() - out64).abs() <= 2 * U * out64.abs().max()).all())
        out.backward(dout)
        assert q_w.grad is None and k_w.grad is None
        torch.cuda.synchronize()
        assert torch.equal(leaf.grad[:, :, nh + nkv:], dout[:, :, nh + nkv:])
        derr = (leaf.grad[:, :, :nh + nkv].double() - dx64).abs()
        assert bool((derr <= U * dx64.abs() + 1e-5 * dx_mag + 1e-38).all())
        err = (flat.double() - want).abs()
        assert bool((err <= tol + U * want.abs()).all()), f"micro-batch {mb}: worst {(err / tol).max().item():.3g}"
    assert q_w._dtg_writes == 2 and k_w._dtg_writes == 2


def test_full_width_binding_refuses_bad_arguments_without_launch():
    C = _C()
    B, S, nh, nkv = 1, 16, 4, 2
    qkv = torch.zeros(B, S, nh + 2 * nkv, 128, device="cuda", dtype=torch.bfloat16)
    qw = torch.ones(nh * 128, device="cuda", dtype=torch.bfloat16)
    kw = torch.ones(nkv * 128, device="cuda", dtype=torch.bfloat16)
    cos, sin = ref.rope_tables(torch.arange(S, device="cuda"), 128, 5e5)
    wide = torch.zeros(B, S, 100 + 2 * 1, 128, device="cuda", dtype=torch.bfloat16)   # 100 + 1 q|k heads
    bad = [
        (dict(qkv=qkv.float()), "qkv"),
        (dict(qkv=torch.zeros(B, S, nh + 2 * nkv, 64, device="cuda", dtype=torch.bfloat16),
              cos=cos[:, :32].contiguous(), sin=sin[:, :32].contiguous()), "head_dim"),
        (dict(qkv=torch.zeros(B, S, nh + 2 * nkv, 256, device="cuda", dtype=torch.bfloat16)[..., :128]), "qkv"),
        (dict(q_w=torch.ones(128, device="cuda", dtype=torch.bfloat16)), "q_w"),   # a per-head gain
        (dict(k_w=torch.ones(nh * 128, device="cuda", dtype=torch.bfloat16)), "k_w"),
        (dict(q_w=qw.float()), "q_w"),
        (dict(k_w=torch.ones(2 * nkv * 128, device="cuda", dtype=torch.bfloat16)[::2]), "k_w"),
        (dict(cos=cos[:15].contiguous(), sin=sin[:15].contiguous()), "neither"),
        (dict(cos=cos.double()), "cos"),
        (dict(sin=sin[:, :32].contiguous()), "sin"),
        (dict(nkv=3), "heads"),
        (dict(eps=float("nan")), "eps"),
        (dict(qkv=wide, nh=100, nkv=1, q_w=torch.ones(100 * 128, device="cuda", dtype=torch.bfloat16),
              k_w=torch.ones(128, device="cuda", dtype=torch.bfloat16)), "q \\+ k heads"),
    ]
    for over, match in bad:
        a = dict(qkv=qkv, q_w=qw, k_w=kw, cos=cos, sin=sin, nh=nh, nkv=nkv, eps=EPS)
        a.update(over)
        n0 = C.launch_count()
        with pytest.raises(RuntimeError, match=match):
            C.qk_norm_full_rope_fwd(a["qkv"], a["q_w"], a["k_w"], a["cos"], a["sin"], a["nh"], a["nkv"], a["eps"])
        assert C.launch_count() == n0, over
    x_save, rstd = C.qk_norm_full_rope_fwd(qkv.clone(), qw, kw, cos, sin, nh, nkv, EPS)
    n0 = C.launch_count()
    with pytest.raises(RuntimeError, match="rstd"):
        C.qk_norm_full_rope_bwd(qkv.clone(), x_save, rstd[:, :, :1].contiguous(), qw, kw, cos, sin, nh, nkv)
    with pytest.raises(RuntimeError, match="x_save"):
        C.qk_norm_full_rope_bwd(qkv.clone(), x_save[:, :, :-1].contiguous(), rstd, qw, kw, cos, sin, nh, nkv)
    with pytest.raises(RuntimeError, match="k_w"):
        C.qk_norm_full_rope_bwd(qkv.clone(), x_save, rstd, qw, qw, cos, sin, nh, nkv)
    assert C.launch_count() == n0
    # the per-token [T, 64] and [B, S, 64] tables are both accepted
    pos = torch.arange(S, device="cuda")[None].expand(2, S)
    c3, s3 = ref.rope_tables(pos, 128, 5e5)
    q2 = torch.zeros(2, S, nh + 2 * nkv, 128, device="cuda", dtype=torch.bfloat16)
    C.qk_norm_full_rope_fwd(q2, qw, kw, c3, s3, nh, nkv, EPS)
    C.qk_norm_full_rope_fwd(q2, qw, kw, c3.reshape(2 * S, 64).contiguous(), s3.reshape(2 * S, 64).contiguous(), nh, nkv,
                            EPS)


# ------------------------------------------------------------------------------------------------------------------
# norm-then-add
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("T,H", [(37, 512), (256, 2048), (131, 4096), (1000, 5120), (64, 8192), (33, 16384)])
def test_norm_then_add_is_rmsnorm_then_bf16_add(T, H):
    """Every hidden-size instantiation: bit-identical to rmsnorm_fwd followed by a bf16 add, same rstd, and within two
    bf16 roundings of fp64."""
    gen = torch.Generator(device="cuda").manual_seed(H)
    x = (torch.randn(T, H, generator=gen, device="cuda") * 3).to(torch.bfloat16)
    x[1] = 0   # an all-zero row
    r = torch.randn(T, H, generator=gen, device="cuda").to(torch.bfloat16)
    w = torch.randn(H, generator=gen, device="cuda").to(torch.bfloat16)
    w[::7] = 0
    C = _C()
    h, rstd = C.rmsnorm_add_fwd(x, r, w, EPS)
    y, rstd_ref, _ = C.rmsnorm_fwd(x, w, EPS, None)
    torch.cuda.synchronize()
    assert torch.equal(h, r + y), "norm-then-add differs from rmsnorm_fwd + a bf16 add"
    assert torch.equal(rstd, rstd_ref)
    xd = x.double()
    y64 = w.double() * xd / torch.sqrt(xd.square().mean(-1, keepdim=True) + EPS)
    h64 = r.double() + y64
    err = (h.double() - h64).abs()
    bound = U * (1 + 1e-5) * y64.abs() + U * h64.abs() + 1e-5 * U * y64.abs() + 1e-38
    assert bool((err <= bound).all()), f"{int((err > bound).sum())} elements off, worst {(err / bound).max():.3g}"


def test_norm_then_add_backward_matches_reference():
    T, H = 300, 4096
    gen = torch.Generator(device="cuda").manual_seed(1)
    x = (torch.randn(T, H, generator=gen, device="cuda") * 2).to(torch.bfloat16)
    r = torch.randn(T, H, generator=gen, device="cuda").to(torch.bfloat16)
    w = torch.randn(H, generator=gen, device="cuda").to(torch.bfloat16)
    dh = torch.randn(T, H, generator=gen, device="cuda").to(torch.bfloat16)
    xl, rl, wl = (t.clone().requires_grad_(True) for t in (x, r, w))
    h = ops.rms_norm_add(xl, rl, wl, EPS)
    h.backward(dh)
    xd, rd, wd = (t.double().requires_grad_(True) for t in (x, r, w))
    ref.rms_norm_add(xd, rd, wd, EPS).backward(dh.double())
    assert torch.equal(rl.grad, dh), "dr must be dh"
    for name, got, want in (("dx", xl.grad, xd.grad), ("dw", wl.grad, wd.grad)):
        rel = ((got.double() - want).norm() / want.norm()).item()
        assert rel < 4e-3, (name, rel)
    # element by element for dx: one bf16 rounding plus fp32 error
    xh = xd.detach() * torch.rsqrt(xd.detach().square().mean(-1, keepdim=True) + EPS)
    g = dh.double() * w.double()
    mag = torch.rsqrt(xd.detach().square().mean(-1, keepdim=True) + EPS) * (
        g.abs() + xh.abs() * (g * xh).abs().mean(-1, keepdim=True))
    assert bool(((xl.grad.double() - xd.grad).abs() <= U * xd.grad.abs() + 1e-5 * mag + 1e-38).all())


def test_norm_then_add_binding_refuses_bad_arguments_without_launch():
    C = _C()
    x = torch.zeros(8, 256, device="cuda", dtype=torch.bfloat16)
    w = torch.ones(256, device="cuda", dtype=torch.bfloat16)
    bad = [
        (dict(x=x.float()), "x"),
        (dict(r=x[:, :128]), "r"),
        (dict(r=torch.zeros(4, 256, device="cuda", dtype=torch.bfloat16)), "shape"),
        (dict(w=torch.ones(128, device="cuda", dtype=torch.bfloat16)), "w"),
        (dict(x=torch.zeros(8, 100, device="cuda", dtype=torch.bfloat16),
              r=torch.zeros(8, 100, device="cuda", dtype=torch.bfloat16),
              w=torch.ones(100, device="cuda", dtype=torch.bfloat16)), "multiple of 8"),
        (dict(eps=-1.0), "eps"),
    ]
    for over, match in bad:
        a = dict(x=x, r=x, w=w, eps=EPS)
        a.update(over)
        n0 = C.launch_count()
        with pytest.raises(RuntimeError, match=match):
            C.rmsnorm_add_fwd(a["x"], a["r"], a["w"], a["eps"])
        assert C.launch_count() == n0, over


# ------------------------------------------------------------------------------------------------------------------
# training steps
# ------------------------------------------------------------------------------------------------------------------
CONFIGS = {
    "olmo2-b2-s256": dict(model="debug-olmo2", B=2, S=256, overrides={}),
    "olmo2-b2-s256-tied": dict(model="debug-olmo2", B=2, S=256, overrides=dict(tie_word_embeddings=True)),
}


@pytest.mark.parametrize("case", list(CONFIGS))
def test_olmo2_step_matches_fp32_reference(case, monkeypatch):
    cfg = CONFIGS[case]
    report, worst = [], 0.0
    with _engine(monkeypatch, cfg) as eng:
        config = eng.config
        assert config.full_qk_norm and config.post_norm
        rec = _capture_buckets(eng)
        for step in (1, 2, 3):
            batch = eng.synthetic_batch(seed=step - 1)
            weights = {n: p.detach().clone() for n, p in eng.model.named_parameters()}
            for key in ("q_norm", "k_norm", "post_feedforward_layernorm"):
                assert any(key in n for n in weights), key
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


def test_olmo2_packed_step_matches_fp32_reference(monkeypatch):
    """Per-token RoPE tables from ``position_ids`` reach the full-width kernel; attention stays inside documents."""
    from distributed_training_guide_b200.engine import TrainEngine

    B, S = 2, 512
    eng = TrainEngine.create("debug-olmo2", parallelism="single", batch_size=B, seq_length=S, lr=5e-3, device="cuda",
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
    _print_report("olmo2 packed step", report)


CHAPTER_ARGS = ["-d", "synthetic", "-m", "debug-olmo2", "-s", "256", "-b", "2", "--num-samples", "32", "--log-freq",
                "1", "-e", "exp", "--lr", "1e-3", "--ckpt-freq", "3"]


def _losses(recs):
    return [r["running_loss"] for r in sorted(recs, key=lambda r: r["global_step"])]


@pytest.mark.parametrize("extra", [[], ["--fp8"]])
def test_chapter01_olmo2_on_gpu_with_resume(tmp_path, extra):
    script = ROOT / "01-single-gpu" / "train_llm.py"
    args = CHAPTER_ARGS + ["--save-dir", str(tmp_path)] + extra
    recs, _ = _run(script, args + ["--max-steps", "3"])
    assert len(recs) == 3 and all(r["tokens_per_s"] > 0 for r in recs)
    assert all(0 < l < 20 and math.isfinite(l) for l in _losses(recs))
    assert json.loads((tmp_path / "exp" / "state.json").read_text())["global_step"] == 3
    recs2, log = _run(script, args + ["--max-steps", "6"])
    assert "Resumed=True" in log and recs2[-1]["global_step"] == 6
    assert all(0 < l < 20 and math.isfinite(l) for l in _losses(recs2))


@pytest.mark.multigpu
@pytest.mark.parametrize("chapter", ["02-distributed-data-parallel", "04-fully-sharded-data-parallel"])
def test_distributed_chapters_olmo2_match_single_gpu(tmp_path, chapter):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    args = [a for a in CHAPTER_ARGS] + ["--max-steps", "4"]
    single, _ = _run(ROOT / "01-single-gpu" / "train_llm.py", args + ["--save-dir", str(tmp_path / "one")])
    recs, _ = _run(ROOT / chapter / "train_llm.py", args + ["--save-dir", str(tmp_path / "many")], nproc=2)
    a, b = _losses(single), _losses(recs)
    # random tokens from the same initial weights: the first losses agree closely, and training stays finite
    assert abs(a[0] - b[0]) < 5e-2, (a, b)
    assert all(math.isfinite(x) and x < a[0] + 0.5 for x in b), (a, b)
