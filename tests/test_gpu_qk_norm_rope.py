"""The QK-norm + RoPE kernels (``csrc/rope.cu``) against an fp64 composition, element by element.

Forward: each output element may differ from the exact ``rope(rmsnorm(x) * w)`` by the three bf16 roundings the
kernel makes (``bf16(x * rstd)``, ``bf16(. * w)``, the stored output): 3 * 2^-8 of the terms the rotation sums.
Backward: ``dx`` is stored once in bf16 after fp32 arithmetic on exact bf16 inputs, so its bound is one bf16
rounding of dx plus fp32 error on the terms ``rstd * (|g| + |xhat| * mean|g * xhat|)``.  The gain gradients are fp32
sums over every token and head, judged relative to the sum of the magnitudes of their terms.

Structure, bit for bit: V (forward) and dV (backward) come back unchanged, the gain gradients are identical across
two runs, and in a flat buffer the first micro-batch overwrites the gain gradients and the second accumulates."""
import math

import pytest
import torch

from distributed_training_guide_b200 import _ext, ops
from distributed_training_guide_b200.ops import reference as ref

pytestmark = pytest.mark.gpu

EPS = 1e-6
U = 2.0 ** -8   # bf16 unit roundoff: rounding to bf16 changes a value by at most U times its magnitude


def _C():
    return _ext.load(required=True)


def _tables(B, S, per_token, gen):
    pos = torch.randint(0, 40960, (B, S), generator=gen, device="cuda") if per_token else torch.arange(S, device="cuda")
    return ref.rope_tables(pos, 128, 1e6)


def _rope64(x, cos, sin, inverse=False):
    c, s = cos.double(), sin.double()
    if c.dim() == 2:
        c, s = c[None, :, None, :], s[None, :, None, :]
    else:
        c, s = c[:, :, None, :], s[:, :, None, :]
    if inverse:
        s = -s
    x1, x2 = x[..., :64], x[..., 64:]
    return torch.cat([x1 * c - x2 * s, x2 * c + x1 * s], dim=-1), (x1.abs() * c.abs() + x2.abs() * s.abs(),
                                                                      x2.abs() * c.abs() + x1.abs() * s.abs())


def _fp64(qkv, q_w, k_w, cos, sin, nh, nkv, dout):
    x = qkv[:, :, :nh + nkv].double()
    w = torch.cat([q_w.double()[None].expand(nh, 128), k_w.double()[None].expand(nkv, 128)])   # [nh+nkv, 128]
    rstd = 1.0 / torch.sqrt(x.square().mean(-1, keepdim=True) + EPS)
    xh = x * rstd
    y = xh * w
    out, (mag1, mag2) = _rope64(y, cos, sin)
    d, _ = _rope64(dout[:, :, :nh + nkv].double(), cos, sin, inverse=True)
    g = d * w
    dot = (g * xh).mean(-1, keepdim=True)
    dx = rstd * (g - xh * dot)
    dx_mag = rstd * (g.abs() + xh.abs() * (g * xh).abs().mean(-1, keepdim=True))
    dwq = (d * xh)[:, :, :nh].sum((0, 1, 2))
    dwk = (d * xh)[:, :, nh:].sum((0, 1, 2))
    mq = (d * xh).abs()[:, :, :nh].sum((0, 1, 2))
    mk = (d * xh).abs()[:, :, nh:].sum((0, 1, 2))
    return out, torch.cat([mag1, mag2], -1), dx, dx_mag, (dwq, dwk), (mq, mk)


def _case(B, S, nh, nkv, per_token, seed, scale=1.0, zero_head=False, gains="random", bf16_max=False):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    qkv = (torch.randn(B, S, nh + 2 * nkv, 128, generator=gen, device="cuda") * scale).to(torch.bfloat16)
    if zero_head:
        qkv[:, 1, 0] = 0
        qkv[:, -1, nh] = 0
    if bf16_max:   # a q head with two and a k head with three elements at the bf16 limit, ordinary heads beside them
        big = torch.finfo(torch.bfloat16).max
        qkv[:, :, 0, 0], qkv[:, :, 0, 64] = big, -big
        qkv[:, :, nh, 3], qkv[:, :, nh, 77], qkv[:, :, nh, 100] = big, big, -big
    q_w = torch.randn(128, generator=gen, device="cuda").to(torch.bfloat16)
    k_w = torch.randn(128, generator=gen, device="cuda").to(torch.bfloat16)
    if gains == "zeros-and-negatives":
        q_w[::5] = 0
        k_w[3::7] = 0
        q_w[1::3] = -q_w[1::3].abs()
        k_w[::2] = -k_w[::2].abs()
    cos, sin = _tables(B, S, per_token, gen)
    dout = torch.randn(B, S, nh + 2 * nkv, 128, generator=gen, device="cuda").to(torch.bfloat16)
    return qkv, q_w, k_w, cos, sin, dout


CASES = {
    # T = 3 * 77 = 231 tokens: not a multiple of any tile, groups past the end of the last warp trip
    "qwen3-8b-heads-ragged": dict(B=3, S=77, nh=32, nkv=8, per_token=False),
    "tp-rank-share-4-1": dict(B=2, S=133, nh=4, nkv=1, per_token=False),
    "mha-16-16-per-token": dict(B=2, S=96, nh=16, nkv=16, per_token=True),
    "gains-zero-negative-per-token": dict(B=1, S=300, nh=4, nkv=1, per_token=True, gains="zeros-and-negatives"),
    "all-zero-heads": dict(B=2, S=64, nh=8, nkv=2, per_token=False, zero_head=True),
    "near-bf16-limit": dict(B=1, S=40, nh=4, nkv=1, per_token=False, scale=1e37),
    # squares whose fp32 sum overflows unless the head is summed scaled down far enough
    "bf16-max-elements": dict(B=2, S=48, nh=4, nkv=2, per_token=False, bf16_max=True),
    "tiny-inputs": dict(B=1, S=40, nh=4, nkv=1, per_token=False, scale=1e-30),
    "long-qwen3-8b": dict(B=1, S=4096, nh=32, nkv=8, per_token=False),
}


@pytest.mark.parametrize("case", list(CASES))
def test_kernels_against_fp64(case):
    c = dict(CASES[case])
    B, S, nh, nkv, per_token = c.pop("B"), c.pop("S"), c.pop("nh"), c.pop("nkv"), c.pop("per_token")
    qkv, q_w, k_w, cos, sin, dout = _case(B, S, nh, nkv, per_token, seed=len(case), **c)
    assert torch.isfinite(qkv.float()).all()
    out64, mag, dx64, dx_mag, (dwq64, dwk64), (mq, mk) = _fp64(qkv, q_w, k_w, cos, sin, nh, nkv, dout)
    C = _C()
    x = qkv.clone()
    x_save, rstd = C.qk_norm_rope_fwd(x, q_w, k_w, cos, sin, nh, nkv, EPS)
    torch.cuda.synchronize()
    assert torch.equal(x[:, :, nh + nkv:], qkv[:, :, nh + nkv:]), "V heads changed"
    assert torch.equal(x_save, qkv[:, :, :nh + nkv]), "the saved pre-norm heads differ from the input"
    got = x[:, :, :nh + nkv].double()
    err = (got - out64).abs()
    # three bf16 roundings on terms of the size of |y|, plus fp32 noise
    bound = 3 * U * (1 + 1e-5) * mag + 1e-38
    assert bool((err <= bound).all()), f"forward: {int((err > bound).sum())} elements off, worst " \
                                       f"{(err / bound).max().item():.3g} of the bound"
    if c.get("zero_head"):
        assert torch.equal(x[:, 1, 0], torch.zeros_like(x[:, 1, 0]))
        torch.testing.assert_close(rstd[:, 1, 0].double(), torch.full_like(rstd[:, 1, 0].double(), 1 / math.sqrt(EPS)),
                                   rtol=1e-6, atol=0)

    d = dout.clone()
    dw = C.qk_norm_rope_bwd(d, x_save, rstd, q_w, k_w, cos, sin, nh, nkv)
    torch.cuda.synchronize()
    assert torch.equal(d[:, :, nh + nkv:], dout[:, :, nh + nkv:]), "dV changed"
    dgot = d[:, :, :nh + nkv].double()
    derr = (dgot - dx64).abs()
    dbound = U * dx64.abs() + 1e-5 * dx_mag + 1e-38
    assert bool((derr <= dbound).all()), f"dx: {int((derr > dbound).sum())} elements off, worst " \
                                         f"{(derr / dbound).max().item():.3g} of the bound"
    for name, got_w, want, m in (("dw_q", dw[0], dwq64, mq), ("dw_k", dw[1], dwk64, mk)):
        werr = (got_w.double() - want).abs()
        wbound = 1e-5 * m + 1e-38
        assert bool((werr <= wbound).all()), f"{name}: worst {(werr / wbound).max().item():.3g} of the bound"
    # the same backward again: bit-identical gain gradients (fixed-order reduction, no atomics)
    d2 = dout.clone()
    dw2 = C.qk_norm_rope_bwd(d2, x_save, rstd, q_w, k_w, cos, sin, nh, nkv)
    assert torch.equal(dw, dw2) and torch.equal(d, d2)


def test_op_matches_kernels_and_accumulates_in_flat_buffers():
    """``ops.qk_norm_rope_`` through autograd with the gains carrying flat-gradient views, as the engines run it:
    the first micro-batch overwrites stale gradient contents, the second accumulates."""
    B, S, nh, nkv = 2, 128, 8, 2
    q_w = torch.nn.Parameter(torch.randn(128, device="cuda").to(torch.bfloat16))
    k_w = torch.nn.Parameter(torch.randn(128, device="cuda").to(torch.bfloat16))
    flat = torch.full((256,), 123.0, device="cuda", dtype=torch.bfloat16)   # stale contents
    q_w._dtg_grad, k_w._dtg_grad = flat[:128], flat[128:]
    q_w._dtg_writes = k_w._dtg_writes = 0
    want = torch.zeros(2, 128, dtype=torch.float64, device="cuda")
    tol = torch.zeros_like(want)
    for mb in range(2):
        qkv, _, _, cos, sin, dout = _case(B, S, nh, nkv, False, seed=10 + mb)
        _, _, _, _, (dwq, dwk), (mq, mk) = _fp64(qkv, q_w.detach(), k_w.detach(), cos, sin, nh, nkv, dout)
        want += torch.stack([dwq, dwk])
        # one bf16 rounding per write of the running sum, fp32 noise on the terms
        tol += U * torch.stack([dwq, dwk]).abs() + 1e-5 * torch.stack([mq, mk])
        leaf = qkv.clone().requires_grad_(True)
        out = ops.qk_norm_rope_(leaf * 1, q_w, k_w, cos, sin, nh, nkv, EPS)
        out.backward(dout)
        assert q_w.grad is None and k_w.grad is None
        torch.cuda.synchronize()
        assert torch.equal(leaf.grad[:, :, nh + nkv:], dout[:, :, nh + nkv:])
        err = (flat.view(2, 128).double() - want).abs()
        assert bool((err <= tol + U * want.abs()).all()), f"micro-batch {mb}: worst {(err / tol).max().item():.3g}"
    assert q_w._dtg_writes == 2 and k_w._dtg_writes == 2


def test_binding_refuses_bad_arguments_without_launch():
    C = _C()
    B, S, nh, nkv = 1, 16, 4, 2
    qkv = torch.zeros(B, S, nh + 2 * nkv, 128, device="cuda", dtype=torch.bfloat16)
    w = torch.ones(128, device="cuda", dtype=torch.bfloat16)
    cos, sin = ref.rope_tables(torch.arange(S, device="cuda"), 128, 1e6)
    bad = [
        (dict(qkv=qkv.float()), "qkv"),
        (dict(qkv=torch.zeros(B, S, nh + 2 * nkv, 64, device="cuda", dtype=torch.bfloat16),
              cos=cos[:, :32].contiguous(), sin=sin[:, :32].contiguous()), "head_dim"),
        (dict(q_w=torch.ones(64, device="cuda", dtype=torch.bfloat16)), "q_w"),
        (dict(k_w=torch.ones(1, 128, device="cuda", dtype=torch.bfloat16)), "k_w"),
        (dict(q_w=w.float()), "q_w"),
        (dict(cos=cos[:15].contiguous(), sin=sin[:15].contiguous()), "neither"),
        (dict(nkv=3), "heads"),
        (dict(nh=0), "heads"),
        (dict(eps=-1.0), "eps"),
    ]
    for over, match in bad:
        a = dict(qkv=qkv, q_w=w, k_w=w, cos=cos, sin=sin, nh=nh, nkv=nkv, eps=EPS)
        a.update(over)
        n0 = C.launch_count()
        with pytest.raises(RuntimeError, match=match):
            C.qk_norm_rope_fwd(a["qkv"], a["q_w"], a["k_w"], a["cos"], a["sin"], a["nh"], a["nkv"], a["eps"])
        assert C.launch_count() == n0, over
    # backward: a wrong rstd / x_save is refused
    x_save, rstd = C.qk_norm_rope_fwd(qkv.clone(), w, w, cos, sin, nh, nkv, EPS)
    n0 = C.launch_count()
    with pytest.raises(RuntimeError, match="rstd"):
        C.qk_norm_rope_bwd(qkv.clone(), x_save, rstd[:, :, :-1].contiguous(), w, w, cos, sin, nh, nkv)
    with pytest.raises(RuntimeError, match="x_save"):
        C.qk_norm_rope_bwd(qkv.clone(), x_save[:, :, :-1].contiguous(), rstd, w, w, cos, sin, nh, nkv)
    assert C.launch_count() == n0
    # the per-token [T, 64] and [B, S, 64] tables are both accepted
    pos = torch.arange(S, device="cuda")[None].expand(2, S)
    c3, s3 = ref.rope_tables(pos, 128, 1e6)
    q2 = torch.zeros(2, S, nh + 2 * nkv, 128, device="cuda", dtype=torch.bfloat16)
    C.qk_norm_rope_fwd(q2, w, w, c3, s3, nh, nkv, EPS)
    C.qk_norm_rope_fwd(q2, w, w, c3.reshape(2 * S, 64).contiguous(), s3.reshape(2 * S, 64).contiguous(), nh, nkv, EPS)
