"""The bf16 wgmma GEMM (mode 0, every operand layout, the 1-CTA and the 2-CTA variant) against the fp64 product.

Two bounds, neither with an outlier budget:
- worst 128 x 256 tile: the relative L2 error of the worst output tile may be at most ``TILE_FACTOR`` times cuBLAS's
  (``torch.matmul`` in bf16 without reduced-precision reductions) on the same operands, plus ``TILE_SLACK``;
- every element: ``|got - exact| <= 2^-8 |exact| + ELEM_C * K * 2^-24 * (|A| @ |B|)``.  The first term is the bf16
  rounding of the output, the second the fp32 accumulation.  This is the bound that sees a single wrong element.

Operands of the edge shapes are views into buffers whose extra rows and columns are NaN, so a read past a logical
extent turns into NaN in C; the output is a view inside a buffer whose bits outside the view must not change, and in
overwrite mode the view starts out NaN, so an element the kernel does not write shows up.
"""
import contextlib

import pytest
import torch

from distributed_training_guide_b200 import _ext
from test_gpu_fp8 import _worst_tile

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16
LAYOUTS = {"nt": (False, True), "nn": (False, False), "tn": (True, False), "tt": (True, True)}  # (trans_a, trans_b)

# Measured on an H100 80GB HBM3 at a 400 W power limit over every shape and mode of this file:
# - worst tile: the kernel's error equals that of the correctly rounded product (1.000x) on every shape, and is 0.57x
#   (accumulate mode: cuBLAS's bf16 addmm rounds twice) to 1.000x cuBLAS's;
# - every element: the largest c any element needs is 2.8e-3 (accumulate, K 64) and 1.1e-3 on the model shapes.
TILE_FACTOR, TILE_SLACK = 1.01, 1e-5
ELEM_C = 1e-2
CHUNK = 16384   # output columns per fp64 reference chunk (a multiple of the 256-column tile)


def _C():
    return _ext.load(True)


@contextlib.contextmanager
def _no_reduced_precision():
    prev = torch.backends.cuda.matmul.allow_bf16_reduced_precision_reduction
    torch.backends.cuda.matmul.allow_bf16_reduced_precision_reduction = False
    try:
        yield
    finally:
        torch.backends.cuda.matmul.allow_bf16_reduced_precision_reduction = prev


def _randn(shape, seed, std=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (std * torch.randn(*shape, device="cuda", generator=g)).to(BF16)


def _poisoned(t):
    """``t`` as a view into a NaN-filled buffer with two extra rows before and after and 8 / 8+ extra columns before
    and after; the row stride is a multiple of 8 elements and the view starts 16-byte aligned."""
    rows, cols = t.shape
    ld = -(-cols // 8) * 8 + 16
    buf = torch.full((rows + 4, ld), float("nan"), device="cuda", dtype=BF16)
    view = buf[2:2 + rows, 8:8 + cols]
    view.copy_(t)
    return view


def _out_view(M, N, fill):
    """An [M, N] view inside a larger buffer of random bits (the sentinel), filled with ``fill`` (a tensor or NaN)."""
    ld = -(-N // 8) * 8 + 16
    buf = _randn((M + 4, ld), seed=12345)
    view = buf[2:2 + M, 8:8 + N]
    if isinstance(fill, torch.Tensor):
        view.copy_(fill)
    else:
        view.fill_(fill)
    return buf, view


def _outside_unchanged(buf, before, M, N):
    mask = torch.ones_like(buf, dtype=torch.bool)
    mask[2:2 + M, 8:8 + N] = False
    return torch.equal(buf.view(torch.int16)[mask], before.view(torch.int16)[mask])


def _operands(M, N, K, trans_a, trans_b, seed=0):
    """Stored operands: a is [M,K] (or [K,M] when trans_a), b is [K,N] (or [N,K] when trans_b)."""
    a = _randn((K, M) if trans_a else (M, K), seed)
    b = _randn((N, K) if trans_b else (K, N), seed + 1)
    return a, b


def _logical(a, b, trans_a, trans_b):
    return (a.t() if trans_a else a), (b.t() if trans_b else b)


def _evaluate(A, B, outs, old=None):
    """Compare bf16 results of A @ B (+ old) against the fp64 result, CHUNK output columns at a time.  A value of None
    in ``outs`` stands for the correctly rounded result.

    Returns, per name in ``outs``: the worst-tile relative error and the largest element ratio
    ``(|got - exact| - 2^-8 |exact|) / (K 2^-24 (|A| @ |B|))``, the least ``c`` the element bound needs."""
    K, N = B.shape
    Ad = A.double()
    Aa = Ad.abs()
    res = {name: [0.0, float("-inf")] for name in outs}
    for j0 in range(0, N, CHUNK):
        j1 = min(N, j0 + CHUNK)
        Bd = B[:, j0:j1].double()
        exact = Ad @ Bd
        if old is not None:
            exact += old[:, j0:j1].double()
        bound = (Aa @ Bd.abs()).mul_(K * 2.0 ** -24).clamp_min_(1e-300)
        for name, got in outs.items():
            g = exact.to(BF16) if got is None else got[:, j0:j1]
            res[name][0] = max(res[name][0], _worst_tile(g, exact))
            ratio = (g.double() - exact).abs_().sub_(exact.abs().mul_(2.0 ** -8)).div_(bound)
            ratio = torch.where(torch.isnan(ratio), torch.full_like(ratio, float("inf")), ratio)
            res[name][1] = max(res[name][1], ratio.max().item())
        del exact, bound, Bd
    return {name: tuple(v) for name, v in res.items()}


def _check(tag, A, B, got, old=None):
    """The kernel's result ``got`` of A @ B (+ old) against both bounds; cuBLAS computes the same on the same
    operands (``addmm`` in bf16 for accumulate mode)."""
    with _no_reduced_precision():
        cublas = (torch.matmul(A.contiguous(), B.contiguous()) if old is None else
                  torch.addmm(old, A.contiguous(), B.contiguous()))
    ev = _evaluate(A, B, {"kernel": got, "cublas": cublas, "rounded": None}, old)
    del cublas
    tile, c = ev["kernel"]
    cub, rnd = ev["cublas"][0], ev["rounded"][0]
    print(f"\n{tag}: worst tile {tile:.3e}  cuBLAS {cub:.3e} ({tile / max(cub, 1e-30):.3f}x)  "
          f"rounded {rnd:.3e} ({tile / max(rnd, 1e-30):.3f}x)  element c {c:.3g} (cuBLAS {ev['cublas'][1]:.3g})")
    assert torch.isfinite(got).all(), f"{tag}: {int((~torch.isfinite(got)).sum())} non-finite elements"
    assert c <= ELEM_C, f"{tag}: an element needs c = {c:.3g} > {ELEM_C}"
    assert tile <= TILE_FACTOR * cub + TILE_SLACK, f"{tag}: worst tile {tile:.3e} vs cuBLAS {cub:.3e}"


# ------------------------------------------------------------------------------------------------------------------
# edge shapes, poisoned padding, overwrite and accumulate
# ------------------------------------------------------------------------------------------------------------------
# (M, N, K): every M below, at and past one and two 128-row tiles, every K from one 8-element step to a ragged long K,
# and N below, at and past one 256-column tile
EDGE_SHAPES = [
    (1, 8, 8), (8, 16, 16), (64, 248, 40), (127, 256, 56), (128, 264, 64), (129, 8, 72), (255, 16, 120),
    (256, 248, 4104), (257, 264, 8), (1, 264, 4104), (257, 256, 40), (129, 248, 120), (127, 16, 4104),
]


@pytest.mark.parametrize("variant", [1, 2])
@pytest.mark.parametrize("layout", list(LAYOUTS))
@pytest.mark.parametrize("M,N,K", EDGE_SHAPES)
def test_gemm_edges_against_fp64(M, N, K, layout, variant):
    trans_a, trans_b = LAYOUTS[layout]
    a, b = _operands(M, N, K, trans_a, trans_b, seed=M + N + K)
    pa, pb = _poisoned(a), _poisoned(b)
    A, B = _logical(a, b, trans_a, trans_b)
    tag = f"M{M} N{N} K{K} {layout} v{variant}"
    # overwrite into a NaN-filled view
    buf, view = _out_view(M, N, float("nan"))
    before = buf.clone()
    _C().gemm(pa, pb, view, trans_a, trans_b, False, variant)
    assert _outside_unchanged(buf, before, M, N), f"{tag}: overwrite wrote outside its view"
    _check(tag, A, B, view)
    # accumulate onto values of the product's size
    old = _randn((M, N), seed=7, std=max(1.0, K ** 0.5))
    buf, view = _out_view(M, N, old)
    before = buf.clone()
    _C().gemm(pa, pb, view, trans_a, trans_b, True, variant)
    assert _outside_unchanged(buf, before, M, N), f"{tag}: accumulate wrote outside its view"
    _check(tag + " acc", A, B, view, old=old)


# ------------------------------------------------------------------------------------------------------------------
# the training GEMMs of Llama-2-7B at T 4096, in the layout each one runs in
# ------------------------------------------------------------------------------------------------------------------
MODEL_SHAPES = {
    "fwd-qkv": (4096, 12288, 4096, "nt"),          # x @ W^T
    "fwd-down": (4096, 4096, 11008, "nt"),
    "dgrad-qkv": (4096, 4096, 12288, "nn"),        # dy @ W
    "wgrad-gate_up": (22016, 4096, 4096, "tn"),    # dy^T @ x
    "lm_head-fwd-V32000": (4096, 32000, 4096, "nt"),
    "lm_head-fwd-V128256-T2048": (2048, 128256, 4096, "nt"),
    "lm_head-wgrad-V32000": (32000, 4096, 4096, "tn"),
    "wgrad-o-T16384": (4096, 4096, 16384, "tn"),
}


@pytest.mark.parametrize("variant", [1, 2])
@pytest.mark.parametrize("case", list(MODEL_SHAPES))
def test_gemm_model_shapes_against_fp64(case, variant):
    M, N, K, layout = MODEL_SHAPES[case]
    trans_a, trans_b = LAYOUTS[layout]
    a, b = _operands(M, N, K, trans_a, trans_b, seed=3)
    out = torch.empty(M, N, device="cuda", dtype=BF16)
    _C().gemm(a, b, out, trans_a, trans_b, False, variant)
    A, B = _logical(a, b, trans_a, trans_b)
    _check(f"{case} v{variant}", A, B, out)
    del out
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------------------------
# data routing: one NaN in A (B) reaches exactly its row (column) of C
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("variant", [1, 2])
@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_gemm_nan_routing(layout, variant):
    trans_a, trans_b = LAYOUTS[layout]
    M, N, K = 296, 520, 200     # M: a row stride of the [K, M] storage must be a multiple of 8
    for i, j, k in [(0, 0, 0), (M - 1, N - 1, K - 1), (129, 257, 64), (255, 263, 63)]:
        a, b = _operands(M, N, K, trans_a, trans_b, seed=11)
        a[(k, i) if trans_a else (i, k)] = float("nan")
        out = torch.empty(M, N, device="cuda", dtype=BF16)
        _C().gemm(a, b, out, trans_a, trans_b, False, variant)
        bad = ~torch.isfinite(out)
        assert bad[i].all() and int(bad.sum()) == N, f"A[{i},{k}]: {int(bad.sum())} non-finite, want row {i} only"
        a, b = _operands(M, N, K, trans_a, trans_b, seed=11)
        b[(j, k) if trans_b else (k, j)] = float("nan")
        _C().gemm(a, b, out, trans_a, trans_b, False, variant)
        bad = ~torch.isfinite(out)
        assert bad[:, j].all() and int(bad.sum()) == M, f"B[{k},{j}]: {int(bad.sum())} non-finite, want column {j}"


# ------------------------------------------------------------------------------------------------------------------
# determinism: two calls, and every variant, give the same bits
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("layout", list(LAYOUTS))
@pytest.mark.parametrize("M,N,K", [(136, 264, 72), (1000, 1288, 1040), (4096, 4096, 4096)])
def test_gemm_bits_equal_across_calls_and_variants(M, N, K, layout):
    """Each output element is accumulated by the same wgmma sequence in the same K order whichever variant runs; the
    CTA pair only changes where the B tile comes from (multicast from the peer)."""
    trans_a, trans_b = LAYOUTS[layout]
    a, b = _operands(M, N, K, trans_a, trans_b, seed=5)
    outs = {}
    for v in (1, 2, 3, 0, 1, 2):
        out = torch.empty(M, N, device="cuda", dtype=BF16)
        _C().gemm(a, b, out, trans_a, trans_b, False, v)
        if v in outs:
            assert torch.equal(outs[v].view(torch.int16), out.view(torch.int16)), f"variant {v}: two calls differ"
        outs[v] = out
    for v in (2, 3, 0):
        diff = int((outs[v].view(torch.int16) != outs[1].view(torch.int16)).sum())
        assert diff == 0, f"variant {v} differs from variant 1 in {diff} of {M * N} elements"


# ------------------------------------------------------------------------------------------------------------------
# contract
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("variant", [1, 2])
def test_gemm_k0_writes_zeros_or_leaves_c(variant):
    """A product over an empty K (a weight gradient over zero tokens) is zero: overwrite mode writes zeros over the
    view, accumulate mode leaves it as it was; nothing outside the view changes."""
    M, N = 200, 264
    for trans_a, trans_b in LAYOUTS.values():
        a = (torch.empty(0, M, device="cuda", dtype=BF16) if trans_a else
             torch.empty(M, 8, device="cuda", dtype=BF16)[:, :0])
        b = (torch.empty(N, 8, device="cuda", dtype=BF16)[:, :0] if trans_b else
             torch.empty(0, N, device="cuda", dtype=BF16))
        for acc in (False, True):
            buf, view = _out_view(M, N, _randn((M, N), seed=1))
            before = buf.clone()
            _C().gemm(a, b, view, trans_a, trans_b, acc, variant)
            torch.cuda.synchronize()
            assert _outside_unchanged(buf, before, M, N)
            want = before[2:2 + M, 8:8 + N] if acc else torch.zeros(M, N, device="cuda", dtype=BF16)
            assert torch.equal(view.view(torch.int16), want.view(torch.int16)), (trans_a, trans_b, acc)
    # fp8: both operands K-major; N and every row stride a multiple of 16
    Nf = 272
    a8 = torch.zeros(M, 16, device="cuda", dtype=torch.float8_e4m3fn)[:, :0]
    b8 = torch.zeros(Nf, 16, device="cuda", dtype=torch.float8_e4m3fn)[:, :0]
    one = torch.ones(1, device="cuda")
    for acc in (False, True):
        buf = _randn((M + 4, Nf + 32), seed=2)
        view = buf[2:2 + M, 16:16 + Nf]
        before = buf.clone()
        _C().gemm_fp8(a8, b8, view, one, one, acc, variant)
        torch.cuda.synchronize()
        mask = torch.ones_like(buf, dtype=torch.bool)
        mask[2:2 + M, 16:16 + Nf] = False
        assert torch.equal(buf[mask].view(torch.int16), before[mask].view(torch.int16))
        want = before[2:2 + M, 16:16 + Nf] if acc else torch.zeros(M, Nf, device="cuda", dtype=BF16)
        assert torch.equal(view.view(torch.int16), want.view(torch.int16)), ("fp8", acc)


def _refused(call, match):
    torch.cuda.synchronize()
    n0 = _ext.launch_count()
    with pytest.raises(RuntimeError, match=match):
        call()
    assert _ext.launch_count() == n0, "a refused call launched a kernel"


def test_gemm_rejects_bad_shapes_and_misaligned_operands():
    """N % 8, a leading dimension % 8 and an operand that does not start on a 16-byte boundary are refused on the
    host, before any launch.  The misaligned views are contiguous in their last dimension and pass every other check:
    C at element offset 1 would make the epilogue's bf16-pair stores misaligned."""
    M, N, K = 256, 256, 128
    a = torch.randn(M, K + 8, device="cuda").to(BF16)
    b = torch.randn(N, K + 8, device="cuda").to(BF16)
    c = torch.empty(M, N + 8, device="cuda", dtype=BF16)
    C = _C()
    _refused(lambda: C.gemm(a[:, :K], b[:N - 4, :K], c[:, :N - 4], False, True, False, 0), "multiples of 8")
    _refused(lambda: C.gemm(a[:, :K], b[:, :K], torch.empty(M, N + 4, device="cuda", dtype=BF16)[:, :N], False, True,
                            False, 0), "multiples of 8")
    _refused(lambda: C.gemm(torch.empty(M, K + 4, device="cuda", dtype=BF16)[:, :K], b[:, :K], c[:, :N], False, True,
                            False, 0), "multiples of 8")
    for acc in (False, True):
        _refused(lambda: C.gemm(a[:, :K], b[:, :K], c[:, 1:1 + N], False, True, acc, 0), "C must start")
        _refused(lambda: C.gemm(a[:, 1:1 + K], b[:, :K], c[:, :N], False, True, acc, 0), "A must start")
        _refused(lambda: C.gemm(a[:, :K], b[:, 1:1 + K], c[:, :N], False, True, acc, 0), "B must start")
    a8 = torch.zeros(M, K + 16, device="cuda", dtype=torch.float8_e4m3fn)
    b8 = torch.zeros(N, K + 16, device="cuda", dtype=torch.float8_e4m3fn)
    c16 = torch.empty(M, N + 16, device="cuda", dtype=BF16)
    one = torch.ones(1, device="cuda")
    _refused(lambda: C.gemm_fp8(a8[:, :K], b8[:, :K], c16[:, 1:1 + N], one, one, False, 0), "C must start")
    _refused(lambda: C.gemm_fp8(a8[:, 8:8 + K], b8[:, :K], c16[:, :N], one, one, False, 0), "A must start")
    _refused(lambda: C.gemm_fp8(a8[:, :K], b8[:, 8:8 + K], c16[:, :N], one, one, False, 0), "B must start")
