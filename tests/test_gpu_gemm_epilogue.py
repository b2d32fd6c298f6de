"""The GEMM epilogue that stages output tiles in shared memory and writes them with TMA stores (bf16 and fp8, overwrite
and accumulate), where its hazards live:

- many tiles per CTA, so each warpgroup's staging area is refilled many times: a tile stored before it was complete,
  or a stale tile stored again, changes elements of C;
- boxes clipped at M and N, with C a view (row stride > N) inside a buffer whose bits outside the view must not change;
- accumulate mode on the same clipped boxes, where the C boxes are loaded into the staging area first.

Operands are small integers, so every fp32 accumulator is exact and the expected output is exactly the correctly
rounded bf16 of ``C_old + A @ B`` (one rounding, as the kernel does): every element is compared bit for bit.
"""
import pytest
import torch

from distributed_training_guide_b200 import _ext
from test_gpu_gemm_reference import LAYOUTS, _out_view, _outside_unchanged, _poisoned

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16


def _C():
    return _ext.load(True)


def _ints(shape, seed, lo, hi):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randint(lo, hi + 1, shape, device="cuda", generator=g).to(torch.float32)


def _operands(M, N, K, layout, seed):
    """(a, b, op(a) @ op(b) in fp64) with entries in [-2, 2]: |A @ B| <= 4K, exact in fp32 for K <= 2^22."""
    trans_a, trans_b = LAYOUTS[layout]
    A = _ints((M, K), seed, -2, 2)
    B = _ints((K, N), seed + 1, -2, 2)
    a = (A.t() if trans_a else A).contiguous().to(BF16)
    b = (B.t() if trans_b else B).contiguous().to(BF16)
    return a, b, A.double() @ B.double()


def _expected(prod, c_old=None):
    return (prod if c_old is None else prod + c_old.double()).float().to(BF16)


def _check(got, want):
    bad = (got.view(torch.int16) != want.view(torch.int16))
    assert not bad.any(), (f"{int(bad.sum())} of {bad.numel()} elements differ; first at "
                           f"{tuple(int(i) for i in bad.nonzero()[0])}")


# 6144 x 5120 is 480 tiles of 256 x 256 over the 66 CTA pairs (or 960 of 128 x 256 over 132 CTAs): about seven tiles
# per CTA, each with different operands.
@pytest.mark.parametrize("variant", [1, 2])
@pytest.mark.parametrize("layout", ["nt", "nn", "tn"])
@pytest.mark.parametrize("accumulate", [False, True], ids=["overwrite", "accumulate"])
def test_many_tiles_per_cta(layout, variant, accumulate):
    M, N, K = 6144, 5120, 128
    a, b, prod = _operands(M, N, K, layout, seed=10)
    trans_a, trans_b = LAYOUTS[layout]
    if accumulate:
        c_old = _ints((M, N), 12, -64, 64).to(BF16)
        out = c_old.clone()
    else:
        c_old = None
        out = torch.full((M, N), float("nan"), device="cuda", dtype=BF16)
    _C().gemm(a, b, out, trans_a, trans_b, accumulate, variant)
    _check(out, _expected(prod, c_old))


# N: one box, one box and 8 columns, a half and 8 columns, two halves and 8 columns; M: 1 row, one warpgroup and a
# row, a CTA pair and change
CLIPPED = [(1, 8), (65, 72), (129, 136), (300, 200), (300, 264)]


@pytest.mark.parametrize("variant", [1, 2])
@pytest.mark.parametrize("layout", list(LAYOUTS))
@pytest.mark.parametrize("accumulate", [False, True], ids=["overwrite", "accumulate"])
@pytest.mark.parametrize("M,N", CLIPPED)
def test_clipped_boxes_in_view(M, N, layout, variant, accumulate):
    K = 192
    a, b, prod = _operands(M, N, K, layout, seed=20)
    trans_a, trans_b = LAYOUTS[layout]
    c_old = _ints((M, N), 22, -64, 64).to(BF16) if accumulate else None
    buf, view = _out_view(M, N, c_old if accumulate else float("nan"))
    before = buf.clone()
    _C().gemm(_poisoned(a), _poisoned(b), view, trans_a, trans_b, accumulate, variant)
    _check(view, _expected(prod, c_old))
    assert _outside_unchanged(buf, before, M, N), "the GEMM wrote outside the output view"


@pytest.mark.parametrize("variant", [1, 2])
@pytest.mark.parametrize("a_fmt", ["e4m3", "e5m2"])
@pytest.mark.parametrize("accumulate", [False, True], ids=["overwrite", "accumulate"])
@pytest.mark.parametrize("M,N", [(65, 80), (300, 208), (2048, 4112)])
def test_fp8_clipped_boxes_in_view(M, N, a_fmt, variant, accumulate):
    """The fp8 GEMM takes the same epilogue after its dequantisation: power-of-two scales keep it exact."""
    K = 256
    A = _ints((M, K), 30, -2, 2)
    B = _ints((N, K), 31, -2, 2)
    a8 = A.to(torch.float8_e5m2 if a_fmt == "e5m2" else torch.float8_e4m3fn)
    b8 = B.to(torch.float8_e4m3fn)
    sa = torch.tensor([0.5], device="cuda")
    sb = torch.tensor([2.0], device="cuda")
    prod = A.double() @ B.double().t()
    c_old = _ints((M, N), 32, -64, 64).to(BF16) if accumulate else None
    buf, view = _out_view(M, N, c_old if accumulate else float("nan"))
    before = buf.clone()
    _C().gemm_fp8(a8, b8, view, sa, sb, accumulate, variant)
    _check(view, _expected(prod, c_old))
    assert _outside_unchanged(buf, before, M, N), "the GEMM wrote outside the output view"
