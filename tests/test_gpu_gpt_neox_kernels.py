"""GPT-NeoX's kernels: the dual LayerNorm, partial rotary RoPE, exact GELU and the parallel-residual output GEMMs.

  * ``layernorm2_fwd``: ``h`` is bit-identical to ``bf16(x + r)``; ``y1`` and ``y2`` (and mean, rstd) are
    bit-identical to ``layernorm_fwd`` run with (w1, b1) and with (w2, b2), on the overflow-scaled rows too.
  * ``layernorm2_bwd`` against fp64 at every dispatch width (H 512 ... 8192), with ``test_gpu_layernorm_gelu.py``'s
    bounds applied to ``g = dy1 w1 + dy2 w2``; the four parameter gradients within 2e-5 of the sums of their terms'
    magnitudes; bit-identical run to run.
  * Partial RoPE: the rotated slice is bit-identical to the full-width kernel run on a copy of that slice; the other
    elements of each head and the V heads keep their bits; the inverse restores the input to bf16 rounding.
  * Exact GELU on every finite bf16 bit pattern: bit-identical to ATen's CUDA ``F.gelu``; the backward within
    ``U |ref64| + 2^-24 |dy|`` of fp64.
  * ``ops.parallel_out`` against two fp32 linears plus an add, forward and backward, and its fp8 form against it."""
import math

import pytest
import torch
import torch.nn.functional as F

from distributed_training_guide_b200 import _ext, ops
from distributed_training_guide_b200.ops import reference as ref
from test_gpu_layernorm_gelu import EPS, SUB, U, _gains, _ln64, _rows

pytestmark = pytest.mark.gpu


def _C():
    return _ext.load(required=True)


# ---------------------------------------------------------------------------------------------------------------
# dual LayerNorm
# ---------------------------------------------------------------------------------------------------------------
# one H per dispatch width of the backward (1x128, 2x128, 2x256, 2x512 vectors x threads), Pythia's widths among them
CASES = [(37, 512, "random"), (300, 1024, "offset"), (129, 2048, "random"), (1000, 4096, "random"),
         (65, 5120, "random"), (33, 8192, "random"), (17, 2048, "constant"), (9, 4096, "huge"), (5, 8192, "huge")]


@pytest.mark.parametrize("T,H,rows", CASES)
@pytest.mark.parametrize("residual", [False, True])
def test_layernorm2_forward_is_layernorm_fwd_twice(T, H, rows, residual):
    g = torch.Generator().manual_seed(T * 5 + H)
    C = _C()
    x = _rows(T, H, rows, g)
    r = torch.randn(T, H, generator=g).bfloat16().cuda() if residual else None
    if residual and rows in ("huge", "constant"):
        r.zero_()
    w1, b1 = _gains(H, "random", g)
    w2, b2 = _gains(H, "negative", g)
    y1, y2, h, mean, rstd = C.layernorm2_fwd(x, r, w1, b1, w2, b2, EPS)
    if residual:
        assert torch.equal(h, x + r)
    else:
        assert h is None
    for w, b, y in ((w1, b1, y1), (w2, b2, y2)):
        y_ref, _, mean_ref, rstd_ref = C.layernorm_fwd(x, r, w, b, EPS)
        assert torch.equal(y, y_ref) and torch.equal(mean, mean_ref) and torch.equal(rstd, rstd_ref)


@pytest.mark.parametrize("T,H,rows", CASES)
@pytest.mark.parametrize("residual", [False, True])
def test_layernorm2_backward_against_fp64(T, H, rows, residual):
    g = torch.Generator().manual_seed(T * 3 + H)
    C = _C()
    h = _rows(T, H, rows, g)
    w1, b1 = _gains(H, "random", g)
    w2, b2 = _gains(H, "zero" if H == 4096 else "negative", g)
    _, _, _, mean, rstd = C.layernorm2_fwd(h, None, w1, b1, w2, b2, EPS)
    _, xhat, rstd64, xmax = _ln64(h, w1, b1)
    dy1 = torch.randn(T, H, generator=g).bfloat16().cuda()
    dy2 = torch.randn(T, H, generator=g).bfloat16().cuda()
    dres = torch.randn(T, H, generator=g).bfloat16().cuda() if residual else None
    dx, dp = C.layernorm2_bwd(dy1, dy2, h, w1, w2, mean, rstd, dres)
    assert dp.shape == (4, H) and dp.dtype == torch.float32
    gg = dy1.double() * w1.double() + dy2.double() * w2.double()
    mg = gg.mean(-1, keepdim=True)
    mgx = (gg * xhat).mean(-1, keepdim=True)
    dx64 = rstd64 * (gg - mg - xhat * mgx) + (dres.double() if residual else 0)
    bound = U * dx64.abs() + 2e-5 * rstd64 * (gg.abs() + gg.abs().mean(-1, keepdim=True)
                                             + xmax * (gg * xhat).abs().mean(-1, keepdim=True)) + SUB
    err = (dx.double() - dx64).abs()
    assert torch.isfinite(dx).all() and (err <= bound).all(), (err - bound).max()
    for i, dy in enumerate((dy1, dy2)):
        dyd = dy.double()
        assert ((dp[2 * i].double() - (dyd * xhat).sum(0)).abs() <= 2e-5 * (dyd.abs() * xmax).sum(0) + 1e-30).all()
        assert ((dp[2 * i + 1].double() - dyd.sum(0)).abs() <= 2e-5 * dyd.abs().sum(0)).all()
    dx2, dp2 = C.layernorm2_bwd(dy1, dy2, h, w1, w2, mean, rstd, dres)   # no atomics: the same bits
    assert torch.equal(dx, dx2) and torch.equal(dp, dp2)


def test_layer_norm2_op_gradients_route_to_the_parameters():
    g = torch.Generator().manual_seed(2)
    T, H = 256, 2048
    x = torch.randn(T, H, generator=g).bfloat16().cuda().requires_grad_()
    r = torch.randn(T, H, generator=g).bfloat16().cuda().requires_grad_()
    ps = [p.clone().requires_grad_() for p in (*_gains(H, "random", g), *_gains(H, "random", g))]
    y1, y2, h = ops.layer_norm2(x, r, *ps, EPS)
    dy1, dy2, dh = (torch.randn(T, H, generator=g).bfloat16().cuda() for _ in range(3))
    torch.autograd.backward([y1, y2, h], [dy1, dy2, dh])
    xf, rf = x.detach().float().requires_grad_(), r.detach().float().requires_grad_()
    pf = [p.detach().float().requires_grad_() for p in ps]
    hf = (xf + rf).bfloat16().float()
    out = [F.layer_norm(hf, (H,), pf[0], pf[1], EPS), F.layer_norm(hf, (H,), pf[2], pf[3], EPS), hf]
    torch.autograd.backward(out, [dy1.float(), dy2.float(), dh.float()])
    # h = bf16(x + r) is rounded in both, so hf's gradient flows to x and r unchanged
    for got, want in [(x.grad, xf.grad), (r.grad, rf.grad)] + [(p.grad, q.grad) for p, q in zip(ps, pf)]:
        assert ((got.float() - want).norm() / want.norm()).item() < 1e-2


def test_layernorm2_refusals():
    C = _C()
    x = torch.zeros(4, 16384, dtype=torch.bfloat16, device="cuda")
    w = torch.ones(16384, dtype=torch.bfloat16, device="cuda")
    with pytest.raises(RuntimeError, match="<= 8192"):
        C.layernorm2_fwd(x, None, w, w, w, w, EPS)
    x, w = x[:, :1024].contiguous(), w[:1024].contiguous()
    with pytest.raises(RuntimeError, match="b2 must be"):
        C.layernorm2_fwd(x, None, w, w, w, w[:512].contiguous(), EPS)
    with pytest.raises(RuntimeError, match="eps"):
        C.layernorm2_fwd(x, None, w, w, w, w, 0.0)


# ---------------------------------------------------------------------------------------------------------------
# partial rotary RoPE
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d,rot", [(128, 32), (64, 16), (128, 64), (128, 96)])
@pytest.mark.parametrize("per_token", [False, True])
def test_partial_rope_is_the_full_kernel_on_the_slice(d, rot, per_token):
    C = _C()
    g = torch.Generator().manual_seed(d + rot)
    B, S, nh = 2, 384, 6
    n_rot = 4   # 2 q + 2 k heads rotate, 2 v heads do not
    x = torch.randn(B, S, nh, d, generator=g).bfloat16().cuda()
    pos = torch.randint(0, 2048, (B, S), generator=g).cuda() if per_token else torch.arange(S, device="cuda")
    cos, sin = ref.rope_tables(pos, rot, 1e4)
    y = x.clone()
    C.rope_inplace(y, cos, sin, n_rot, False, rot_dim=rot)
    want = x[..., :rot].contiguous()
    C.rope_inplace(want, cos, sin, n_rot, False)   # the full-width kernel on a head of rot elements
    assert torch.equal(y[..., :rot], want)
    assert torch.equal(y[..., rot:], x[..., rot:]) and torch.equal(y[:, :, n_rot:], x[:, :, n_rot:])
    assert not torch.equal(y[:, :, :n_rot, :rot], x[:, :, :n_rot, :rot])
    C.rope_inplace(y, cos, sin, n_rot, True, rot_dim=rot)
    assert torch.equal(y[..., rot:], x[..., rot:])
    # a rotation keeps the length m of each pair (j, j + rot/2); each of the two roundings per element is within
    # U/2 of m, so the round trip is within 2 U m of the input
    xs = x[..., :rot].float()
    m = torch.hypot(xs[..., :rot // 2], xs[..., rot // 2:]).repeat(1, 1, 1, 2)
    assert ((y[..., :rot].float() - xs).abs() <= 2 * U * m + SUB).all()


def test_rope_rot_dim_default_is_the_head_and_refusals():
    C = _C()
    x = torch.randn(1, 128, 4, 128).bfloat16().cuda()
    cos, sin = ref.rope_tables(torch.arange(128, device="cuda"), 128, 1e4)
    a, b = x.clone(), x.clone()
    C.rope_inplace(a, cos, sin, 2, False)
    C.rope_inplace(b, cos, sin, 2, False, rot_dim=128)
    assert torch.equal(a, b)
    c32, s32 = ref.rope_tables(torch.arange(128, device="cuda"), 32, 1e4)
    for rot, match in ((24, "multiple of 16"), (256, "<= head_dim"), (0, "positive")):
        with pytest.raises(RuntimeError, match=match):
            C.rope_inplace(x.clone(), c32, s32, 2, False, rot_dim=rot)
    with pytest.raises(RuntimeError, match="wrong shape"):
        C.rope_inplace(x.clone(), cos, sin, 2, False, rot_dim=32)


# ---------------------------------------------------------------------------------------------------------------
# exact GELU
# ---------------------------------------------------------------------------------------------------------------
def _all_finite_bf16():
    bits = torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16)
    x = bits.view(torch.bfloat16)
    return x[torch.isfinite(x)].cuda()


def test_gelu_forward_bit_identical_to_aten_on_every_finite_bf16():
    C = _C()
    x = _all_finite_bf16()
    n = x.numel() // 8 * 8
    x = x[:n].contiguous()
    y = C.gelu_fwd(x)
    want = F.gelu(x)
    same = (y.view(torch.int16) == want.view(torch.int16))
    assert same.all(), (x[~same][:8], y[~same][:8], want[~same][:8])


def test_gelu_backward_against_fp64():
    C = _C()
    x = _all_finite_bf16()
    n = x.numel() // 8 * 8
    x = x[:n].contiguous()
    dy = torch.randn(n, generator=torch.Generator().manual_seed(3)).bfloat16().cuda()
    dx = C.gelu_bwd(dy, x)
    xd, dyd = x.double(), dy.double()
    cdf = 0.5 * (1 + torch.erf(xd / math.sqrt(2)))
    pdf = torch.exp(-0.5 * xd * xd) / math.sqrt(2 * math.pi)
    pdf = torch.where(torch.isfinite(pdf), pdf, torch.zeros_like(pdf))
    ref64 = dyd * (cdf + torch.nan_to_num(xd * pdf, nan=0.0))
    err = (dx.double() - ref64).abs()
    bound = U * ref64.abs() + 2.0 ** -24 * dyd.abs() + SUB
    assert (err <= bound).all(), (x[err > bound][:8], dx[err > bound][:8], ref64[err > bound][:8])
    # ops.gelu's backward is this kernel: autograd through it equals the binding
    xr = x[:4096].clone().requires_grad_()
    ops.gelu(xr).backward(dy[:4096])
    assert torch.equal(xr.grad, dx[:4096])


# ---------------------------------------------------------------------------------------------------------------
# parallel_out
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fp8", [False, True])
def test_parallel_out_matches_two_linears_plus_an_add(fp8):
    g = torch.Generator().manual_seed(11)
    T, H, I = 512, 1024, 4096

    def rnd(*shape, s=1.0):
        return (torch.randn(*shape, generator=g) * s).bfloat16().cuda().requires_grad_()

    a, m = rnd(2, T // 2, H), rnd(2, T // 2, I)
    wd, w4 = rnd(H, H, s=0.03), rnd(H, I, s=0.015)
    bd, b4 = rnd(H, s=0.1), rnd(H, s=0.1)
    out = ops.parallel_out(a, m, wd, w4, bd, b4, fp8=fp8)
    dy = torch.randn(out.shape, generator=g).bfloat16().cuda()
    out.backward(dy)
    leaves = [t.detach().float().requires_grad_() for t in (a, m, wd, w4, bd, b4)]
    want = F.linear(leaves[0], leaves[2], leaves[4]) + F.linear(leaves[1], leaves[3], leaves[5])
    want.backward(dy.float())
    tol = 0.1 if fp8 else 1e-2
    assert ((out.float() - want).norm() / want.norm()).item() < tol
    for t, w in zip((a, m, wd, w4, bd, b4), leaves):
        assert ((t.grad.float() - w.grad).norm() / w.grad.norm()).item() < tol
    assert torch.equal(bd.grad, b4.grad)   # one column sum feeds both biases
