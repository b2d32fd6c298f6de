"""The LayerNorm and GELU-tanh kernels (StarCoder2's block) element by element against fp64.

Bounds (U = 2^-8, bf16's unit roundoff):
  * LayerNorm forward: ``|y - y64| <= U |y64| + 2e-5 (|h| + max|h|) rstd |w|``: the one rounding to bf16, plus fp32
    error in the row statistics, relative to the magnitudes ``h - mean`` is computed from.  ``h = bf16(x + r)`` is
    exact.  Both bounds add 2^-133, bf16's subnormal spacing, for outputs below 2^-126 (dx of rows near bf16's top,
    whose rstd is about 1e-38).
  * LayerNorm backward: ``|dx - dx64| <= U |dx64| + 2e-5 rstd (|g| + mean|g| + xmax mean|g xhat|)`` with ``g = dy w``
    and ``xmax = (|h| + max|h|) rstd``: one rounding plus fp32 error on the terms of
    ``rstd (g - mean(g) - xhat mean(g xhat))``; ``dw`` and ``db`` within ``2e-5`` of the sums of their terms'
    magnitudes (fp32 partial sums over rows, then over CTAs).  Both are bit-identical run to run.
  * GELU-tanh, every finite bf16 input: equal to ATen's bf16 ``gelu(approximate="tanh")`` (and its autograd
    backward), or within ``U |ref64| + 2^-21 |x|`` (forward; ``1 + tanh`` cancels for negative x) and
    ``U |ref64| + 2^-21 |dy| (1 + |x| (1 + 0.135 x^2))`` (backward; ``1 - tanh^2`` cancels) of fp64.  Where tanh has
    saturated (|x| >= 10, and +-inf) the backward is exactly ``dy`` or 0.
NaN reaches exactly the outputs that depend on it; every binding refusal happens before any launch."""
import math

import pytest
import torch
import torch.nn.functional as F

from distributed_training_guide_b200 import _ext, ops

pytestmark = pytest.mark.gpu

U = 2.0 ** -8
SUB = 2.0 ** -133   # the spacing of bf16's subnormals: below 2^-126 a rounding is absolute, not relative
EPS = 1e-5


def _C():
    return _ext.load(required=True)


def _ln64(h, w, b, eps=EPS):
    hf = h.double()
    mean = hf.mean(-1, keepdim=True)
    var = ((hf - mean) ** 2).mean(-1, keepdim=True)
    rstd = 1.0 / torch.sqrt(var + eps)
    xhat = (hf - mean) * rstd
    xmax = (hf.abs() + hf.abs().amax(-1, keepdim=True)) * rstd
    return xhat * w.double() + b.double(), xhat, rstd, xmax


def _rows(T, H, kind, g):
    dev = "cuda"
    if kind == "random":
        x = torch.randn(T, H, generator=g) * 2 + 0.5
    elif kind == "constant":   # var 0: xhat = 0 and y = b
        x = torch.full((T, H), 1.5)
    elif kind == "huge":       # sums overflow fp32: the scaled path
        x = (torch.rand(T, H, generator=g) * 2 - 1) * 3.0e38
    elif kind == "offset":     # mean far from 0 relative to the spread
        x = torch.randn(T, H, generator=g) + 100.0
    return x.bfloat16().to(dev)


def _gains(H, kind, g):
    w = torch.randn(H, generator=g) * 1.5
    if kind == "zero":
        w[:] = 0
    elif kind == "negative":
        w = -w.abs()
    b = torch.randn(H, generator=g)
    return w.bfloat16().cuda(), b.bfloat16().cuda()


CASES = [(37, 512, "random", "random"), (300, 3072, "random", "negative"), (129, 4608, "offset", "random"),
         (1000, 6144, "random", "zero"), (65, 16384, "random", "random"), (17, 3072, "constant", "random"),
         (33, 4608, "huge", "random"), (5, 16384, "huge", "negative")]


@pytest.mark.parametrize("T,H,rows,gains", CASES)
@pytest.mark.parametrize("residual", [False, True])
def test_layernorm_against_fp64(T, H, rows, gains, residual):
    g = torch.Generator().manual_seed(T * 7 + H)
    C = _C()
    x = _rows(T, H, rows, g)
    r = torch.randn(T, H, generator=g).bfloat16().cuda() if residual else None
    if residual and rows in ("huge", "constant"):   # keep h = x + r at the magnitude / constancy under test
        r.zero_()
    w, b = _gains(H, gains, g)
    y, h, mean, rstd = C.layernorm_fwd(x, r, w, b, EPS)
    if residual:
        assert torch.equal(h, x + r)   # bf16(x + r): one rounding, as ATen's bf16 add
    else:
        assert h is None
        h = x
    y64, xhat, rstd64, xmax = _ln64(h, w, b)
    bound = U * y64.abs() + 2e-5 * xmax * w.double().abs() + SUB
    err = (y.double() - y64).abs()
    assert torch.isfinite(y).all() and (err <= bound).all(), (err - bound).max()
    torch.testing.assert_close(rstd.double(), rstd64[:, 0], rtol=1e-5, atol=0)
    torch.testing.assert_close(mean.double(), h.double().mean(-1), rtol=1e-5, atol=1e-6 * float(h.float().abs().max()))
    if rows == "constant":
        assert torch.equal(y, b.expand_as(y))

    dy = torch.randn(T, H, generator=g).bfloat16().cuda()
    dres = torch.randn(T, H, generator=g).bfloat16().cuda() if residual else None
    dx, dw, db = C.layernorm_bwd(dy, h, w, mean, rstd, dres)
    gg = dy.double() * w.double()
    mg = gg.mean(-1, keepdim=True)
    mgx = (gg * xhat).mean(-1, keepdim=True)
    dx64 = rstd64 * (gg - mg - xhat * mgx) + (dres.double() if residual else 0)
    bound = U * dx64.abs() + 2e-5 * rstd64 * (gg.abs() + gg.abs().mean(-1, keepdim=True)
                                             + xmax * (gg * xhat).abs().mean(-1, keepdim=True)) + SUB
    err = (dx.double() - dx64).abs()
    assert (err <= bound).all(), (err - bound).max()
    dyd = dy.double()
    assert ((dw.double() - (dyd * xhat).sum(0)).abs() <= 2e-5 * (dyd.abs() * xmax).sum(0) + 1e-30).all()
    assert ((db.double() - dyd.sum(0)).abs() <= 2e-5 * dyd.abs().sum(0)).all()
    # no atomics: the same inputs give the same bits
    dx2, dw2, db2 = C.layernorm_bwd(dy, h, w, mean, rstd, dres)
    assert torch.equal(dx, dx2) and torch.equal(dw, dw2) and torch.equal(db, db2)


def test_layernorm_nan_reaches_exactly_its_dependents():
    C = _C()
    g = torch.Generator().manual_seed(1)
    T, H = 64, 3072
    x = torch.randn(T, H, generator=g).bfloat16().cuda()
    w, b = _gains(H, "random", g)
    x[5, 17] = float("nan")
    y, _, mean, rstd = C.layernorm_fwd(x, None, w, b, EPS)
    assert torch.isnan(y[5]).all() and torch.isnan(mean[5]) and torch.isnan(rstd[5])
    keep = torch.ones(T, dtype=torch.bool)
    keep[5] = False
    assert torch.isfinite(y[keep]).all() and torch.isfinite(mean[keep]).all()
    # a NaN in dy at (9, 40): row 9 of dx, column 40 of dw and db; nothing else
    x[5, 17] = 0.0
    y, _, mean, rstd = C.layernorm_fwd(x, None, w, b, EPS)
    dy = torch.randn(T, H, generator=g).bfloat16().cuda()
    dy[9, 40] = float("nan")
    dx, dw, db = C.layernorm_bwd(dy, x, w, mean, rstd, None)
    assert torch.isnan(dx[9]).all()
    keep = torch.ones(T, dtype=torch.bool)
    keep[9] = False
    assert torch.isfinite(dx[keep]).all()
    cols = torch.ones(H, dtype=torch.bool)
    cols[40] = False
    assert torch.isnan(dw[40]) and torch.isnan(db[40])
    assert torch.isfinite(dw[cols]).all() and torch.isfinite(db[cols]).all()


def test_layernorm_ops_accumulate_into_flat_buffers():
    """ops.add_layer_norm: the kernel's outputs, and gain / bias gradients overwrite then accumulate."""
    g = torch.Generator().manual_seed(2)
    T, H = 256, 512
    x = torch.randn(2, T // 2, H, generator=g).bfloat16().cuda().requires_grad_()
    r = torch.randn(2, T // 2, H, generator=g).bfloat16().cuda().requires_grad_()
    w = torch.nn.Parameter(torch.randn(H, generator=g).bfloat16().cuda())
    b = torch.nn.Parameter(torch.randn(H, generator=g).bfloat16().cuda())
    flat = torch.zeros(2 * H, dtype=torch.bfloat16, device="cuda")
    w._dtg_grad, b._dtg_grad = flat[:H], flat[H:]
    y, h = ops.add_layer_norm(x, r, w, b, EPS)
    C = _C()
    y_k, h_k, mean, rstd = C.layernorm_fwd(x.detach().reshape(T, H), r.detach().reshape(T, H), w.detach(),
                                           b.detach(), EPS)
    assert torch.equal(y.reshape(T, H), y_k) and torch.equal(h.reshape(T, H), h_k)
    dy = torch.randn(2, T // 2, H, generator=g).bfloat16().cuda()
    dh = torch.randn(2, T // 2, H, generator=g).bfloat16().cuda()
    torch.autograd.backward([y, h], [dy, dh])
    dx_k, dw_k, db_k = C.layernorm_bwd(dy.reshape(T, H), h_k, w.detach(), mean, rstd, dh.reshape(T, H))
    assert torch.equal(x.grad.reshape(T, H), dx_k) and torch.equal(r.grad.reshape(T, H), dx_k)
    assert w.grad is None and torch.equal(flat[:H], dw_k.bfloat16()) and torch.equal(flat[H:], db_k.bfloat16())
    dw_first = flat[:H].clone()
    ops.layer_norm(x.detach(), w, b, EPS).backward(dy)   # a second use in the step: accumulate
    assert torch.equal(flat[H:], db_k.bfloat16() * 2)   # db does not depend on the normalised input
    assert not torch.equal(flat[:H], dw_first)


def _all_bf16():
    bits = torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16)
    x = bits.view(torch.bfloat16).cuda()
    return x[~torch.isnan(x)]


def test_gelu_tanh_over_the_whole_bf16_range():
    C = _C()
    x = _all_bf16()
    x = x[: x.numel() // 8 * 8].contiguous()
    y = C.gelu_tanh_fwd(x)
    ya = F.gelu(x, approximate="tanh")
    xd = x.double()
    fin = torch.isfinite(xd)
    y64 = 0.5 * xd * (1 + torch.tanh(math.sqrt(2 / math.pi) * (xd + 0.044715 * xd ** 3)))
    y64 = torch.where(fin, y64, torch.where(xd > 0, xd, torch.zeros_like(xd)))
    ok = (y == ya) | ((y.double() - y64).abs() <= U * y64.abs() + 2.0 ** -21 * xd.abs().nan_to_num(posinf=0))
    assert ok[fin].all(), x[fin & ~ok][:10]
    # +inf passes through; -inf gives ATen's NaN (0.5 x (1 + tanh) = -inf * 0)
    assert torch.equal(y[~fin & (xd > 0)], x[~fin & (xd > 0)])
    assert torch.isnan(y[~fin & (xd < 0)]).all() and torch.isnan(ya[~fin & (xd < 0)]).all()
    print(f"gelu_tanh forward: {(y == ya).double().mean().item():.5f} of all bf16 inputs bit-identical to ATen")

    dy = torch.randn(x.numel(), generator=torch.Generator().manual_seed(3)).bfloat16().cuda()
    dx = C.gelu_tanh_bwd(dy, x)
    xa = x.clone().requires_grad_()
    F.gelu(xa, approximate="tanh").backward(dy)
    k0, k1 = math.sqrt(2 / math.pi), 0.044715
    t = torch.tanh(k0 * (xd + k1 * xd ** 3))
    d64 = dy.double() * (0.5 * (1 + t) + 0.5 * xd * (1 - t * t) * k0 * (1 + 3 * k1 * xd ** 2))
    big = xd.abs() >= 10
    assert (dx[big] == torch.where(xd[big] > 0, dy[big], torch.zeros_like(dy[big]))).all()
    small = ~big
    bound = U * d64.abs() + 2.0 ** -21 * dy.double().abs() * (1 + xd.abs() * (1 + 0.135 * xd ** 2))
    ok = (dx == xa.grad) | ((dx.double() - d64).abs() <= bound)
    assert ok[small].all(), x[small & ~ok][:10]
    print(f"gelu_tanh backward: {(dx == xa.grad).double().mean().item():.5f} bit-identical to ATen")


def test_gelu_tanh_nan_and_op():
    C = _C()
    x = torch.randn(64, 128, generator=torch.Generator().manual_seed(4)).bfloat16().cuda()
    x[3, 7] = float("nan")
    y = C.gelu_tanh_fwd(x)
    assert torch.isnan(y[3, 7]) and torch.isnan(y).sum() == 1
    dy = torch.ones_like(x)
    dx = C.gelu_tanh_bwd(dy, x)
    assert torch.isnan(dx[3, 7]) and torch.isnan(dx).sum() == 1
    x[3, 7] = 1.0
    dy[10, 10] = float("nan")
    assert torch.isnan(C.gelu_tanh_bwd(dy, x)).sum() == 1
    # the op is the kernel pair
    xa = x.clone().requires_grad_()
    out = ops.gelu_tanh(xa)
    assert torch.equal(out, C.gelu_tanh_fwd(x))
    out.backward(torch.ones_like(x))
    assert torch.equal(xa.grad, C.gelu_tanh_bwd(torch.ones_like(x), x))


def test_bindings_refuse_bad_arguments_without_launch():
    C = _C()
    T, H = 16, 512
    x = torch.randn(T, H, device="cuda").bfloat16()
    w = torch.ones(H, device="cuda", dtype=torch.bfloat16)
    b = torch.zeros(H, device="cuda", dtype=torch.bfloat16)
    y, _, mean, rstd = C.layernorm_fwd(x, None, w, b, EPS)
    torch.cuda.synchronize()
    n0 = C.launch_count()
    misaligned = x.reshape(-1)[1:1 + (T - 1) * H].view(T - 1, H)
    fwd = [
        (lambda: C.layernorm_fwd(x.float(), None, w, b, EPS), "x"),
        (lambda: C.layernorm_fwd(x.t(), None, w, b, EPS), "x"),
        (lambda: C.layernorm_fwd(misaligned, None, w, b, EPS), "x"),
        (lambda: C.layernorm_fwd(x[:, :12].contiguous(), None, w[:12].contiguous(), b[:12].contiguous(), EPS),
         "multiple of 8"),
        (lambda: C.layernorm_fwd(torch.zeros(2, 16392, device="cuda", dtype=torch.bfloat16), None,
                                 torch.ones(16392, device="cuda", dtype=torch.bfloat16),
                                 torch.ones(16392, device="cuda", dtype=torch.bfloat16), EPS), "16384"),
        (lambda: C.layernorm_fwd(x, None, w[:256].contiguous(), b, EPS), "w"),
        (lambda: C.layernorm_fwd(x, None, w.float(), b, EPS), "w"),
        (lambda: C.layernorm_fwd(x, None, w, b[:256].contiguous(), EPS), "b"),
        (lambda: C.layernorm_fwd(x, None, w, b.float(), EPS), "b"),
        (lambda: C.layernorm_fwd(x, x[:8].contiguous(), w, b, EPS), "residual"),
        (lambda: C.layernorm_fwd(x, x.float(), w, b, EPS), "residual"),
        (lambda: C.layernorm_fwd(x, None, w, b, 0.0), "eps"),
        (lambda: C.layernorm_fwd(x, None, w, b, -1e-5), "eps"),
        (lambda: C.layernorm_fwd(x, None, w, b, float("nan")), "eps"),
        (lambda: C.layernorm_fwd(x, None, w, b, float("inf")), "eps"),
        (lambda: C.layernorm_fwd(x[0].contiguous(), None, w, b, EPS), "2-D"),
    ]
    bwd = [
        (lambda: C.layernorm_bwd(x, x[:8].contiguous(), w, mean, rstd, None), "h"),
        (lambda: C.layernorm_bwd(x.float(), x, w, mean, rstd, None), "dy"),
        (lambda: C.layernorm_bwd(x, x, w, mean[:8].contiguous(), rstd, None), "mean"),
        (lambda: C.layernorm_bwd(x, x, w, mean, rstd.half(), None), "rstd"),
        (lambda: C.layernorm_bwd(x, x, w, mean, rstd, x[:8].contiguous()), "dres"),
        (lambda: C.layernorm_bwd(x, x, w[:256].contiguous(), mean, rstd, None), "w"),
    ]
    gelu = [
        (lambda: C.gelu_tanh_fwd(torch.zeros(3, 5, device="cuda", dtype=torch.bfloat16)), "multiple of 8"),
        (lambda: C.gelu_tanh_fwd(x.float()), "x"),
        (lambda: C.gelu_tanh_fwd(x.t()), "x"),
        (lambda: C.gelu_tanh_bwd(x, x[:8].contiguous()), "differ"),
        (lambda: C.gelu_tanh_bwd(x.float(), x), "dy"),
        (lambda: C.gelu_tanh_bwd(x[:T - 1].contiguous(), misaligned), "16-byte aligned"),
    ]
    for fn, msg in fwd + bwd + gelu:
        with pytest.raises(RuntimeError, match=msg):
            fn()
    torch.cuda.synchronize()
    assert C.launch_count() == n0
