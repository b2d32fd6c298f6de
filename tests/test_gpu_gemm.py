"""wgmma GEMM (all operand layouts, 1-CTA and 2-CTA variants) vs an fp32 reference."""
import os

import pytest
import torch

from distributed_training_guide_b200 import _ext, ops

pytestmark = pytest.mark.gpu
DEV = "cuda"

SHAPES = [
    (128, 256, 64),       # one tile, one k-block
    (256, 512, 256),      # 2x2 tiles
    (384, 768, 192),      # odd tile counts, k tail of 3 blocks
    (200, 264, 72),       # ragged M/N/K (masked epilogue, TMA zero fill)
    (4096, 4096, 4096),   # the 7B projection shape
    (1024, 11008, 4096),
]


def _ref(a, b, trans_a, trans_b):
    A = a.float().t() if trans_a else a.float()
    B = b.float().t() if trans_b else b.float()
    return A @ B


@pytest.mark.parametrize("variant", [1, 2])
@pytest.mark.parametrize("trans_a,trans_b", [(False, True), (False, False), (True, False), (True, True)])
@pytest.mark.parametrize("M,N,K", SHAPES)
def test_gemm_layouts(M, N, K, trans_a, trans_b, variant):
    torch.manual_seed(0)
    C = _ext.load(True)
    a = torch.randn((K, M) if trans_a else (M, K), device=DEV, dtype=torch.bfloat16)
    b = torch.randn((N, K) if trans_b else (K, N), device=DEV, dtype=torch.bfloat16)
    out = torch.full((M, N), float("nan"), device=DEV, dtype=torch.bfloat16)
    C.gemm(a, b, out, trans_a, trans_b, False, variant)
    want = _ref(a, b, trans_a, trans_b)
    err = (out.float() - want).abs()
    tol = 0.02 * want.abs() + 0.02 * (K ** 0.5)
    assert torch.isfinite(out.float()).all(), "unwritten / non-finite outputs"
    assert (err <= tol).all(), f"max err {err.max().item():.4g} (K={K})"
    # accumulate: out += a@b
    base = torch.randn(M, N, device=DEV, dtype=torch.bfloat16)
    out2 = base.clone()
    C.gemm(a, b, out2, trans_a, trans_b, True, variant)
    err2 = (out2.float() - (want + base.float())).abs()
    assert (err2 <= tol + 0.02 * base.float().abs() + 0.05).all(), f"accumulate: max err {err2.max().item():.4g}"


def test_gemm_strided_views():
    """Operands that are row-slices / column-slices of larger buffers (fused qkv, flat grads)."""
    torch.manual_seed(0)
    C = _ext.load(True)
    big = torch.randn(512, 1024, device=DEV, dtype=torch.bfloat16)
    a = big[:, 256:768]            # [512, 512], row stride 1024
    w = torch.randn(384, 512, device=DEV, dtype=torch.bfloat16)
    outbuf = torch.zeros(512, 1024, device=DEV, dtype=torch.bfloat16)
    out = outbuf[:, 128:512]
    C.gemm(a, w, out, False, True, False, 0)
    want = a.float() @ w.float().t()
    assert ((out.float() - want).abs() <= 0.02 * want.abs() + 0.5).all()
    assert outbuf[:, :128].abs().sum() == 0 and outbuf[:, 512:].abs().sum() == 0


def test_linear_autograd():
    torch.manual_seed(0)
    x = torch.randn(4, 96, 512, device=DEV, dtype=torch.bfloat16, requires_grad=True)
    w = (0.05 * torch.randn(768, 512, device=DEV)).to(torch.bfloat16).requires_grad_(True)
    y = ops.linear(x, w)
    dy = torch.randn_like(y)
    y.backward(dy)
    xf, wf = x.detach().float().requires_grad_(True), w.detach().float().requires_grad_(True)
    yf = xf @ wf.t()
    yf.backward(dy.float())
    assert ((y.float() - yf).abs() <= 0.02 * yf.abs() + 0.05).all()
    assert ((x.grad.float() - xf.grad).abs() <= 0.02 * xf.grad.abs() + 0.1).all()
    assert ((w.grad.float() - wf.grad).abs() <= 0.02 * wf.grad.abs() + 0.6).all()
