"""The fp8 wgmma GEMM and the fp8 casts against fp64, element by element, at their edges.

The GEMM's contract, with ``deq = fp32(scale_a * scale_b)`` and ``acc`` the accumulator of ``A8 @ B8^T``:
overwrite ``bf16(fp32(acc * deq))``, accumulate ``bf16(fp32(acc * deq + C_old))`` (one rounding), bias
``bf16(fp32(acc * deq + bias))``.

a. Exact designs, every element bit for bit with no tolerance: the accumulator is exact by construction (one product
   per output, or small-integer sums with sum_k |a_k b_k| <= 2^10), so the expected output is fp64 -> fp32 -> bf16.
   Operands are views inside buffers of byte 0x7F (NaN in both e4m3fn and e5m2), so a read past K, M or N turns into
   NaN; the output is a view inside a sentinel buffer whose bits outside the view must not change.
b. Random data at the training shapes, every element against
   ``|got - exact| <= 2^-8 |exact| + ELEM_C * 2^-13 * deq * sum_t (|S_(t-1)| + sum_(k in t) |a_k b_k|)``:
   the first term is the bf16 rounding of the output, the second one truncation to 13 bits per k32 wgmma step t, in
   the kernel's ascending-K order, of a partial sum S_t (the fp64 sum of the first 32 t products) and the step's
   products.  The fp8 wgmma does not accumulate in full fp32, so the bf16 file's n 2^-24 bound does not hold here.
c. Position independence: an element's bits do not depend on its tile, the variant or the output's row stride.
d. NaN / Inf operands, K = 0, M = 0 and N = 0.
e. Every refusal happens on the host, before any launch.
The casts: every finite bf16 value at an amax in every bf16 binade, bit for bit against the reference quantisation
and against fp64.

Measured on an H100 80GB HBM3 at a 700 W power limit:
- fp8 subnormals survive the tensor core: every product of two finite codes, 6916 (e4m3 x e4m3) and 4912
  (e5m2 x e4m3) of them with a subnormal operand, is exact;
- the largest ELEM_C any element needs is 0.554 in overwrite mode and 0.616 in accumulate mode (fwd-qkv), 0.30 to
  0.62 over the shapes, so the 13-bit model holds; the perturbed outputs of the checker's self-test need 3.1 (one
  element by 1 %) and 6.5 (one row by 2 ulps);
- the whole file takes 12 s.
"""
import pytest
import torch

from distributed_training_guide_b200 import _ext
from distributed_training_guide_b200.ops import reference as ref
from test_gpu_fp8 import GEMM_SHAPES, _operands
from test_gpu_gemm_reference import _out_view, _outside_unchanged, _refused

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16
E4M3, E5M2 = torch.float8_e4m3fn, torch.float8_e5m2
FMTS = {"e4m3": E4M3, "e5m2": E5M2}
POISON = 0x7F     # NaN in e4m3fn and in e5m2

# Random data (b): the largest c any element needs is 0.616 (see above); 1 would mean the model is wrong.
ELEM_C = 0.75
CHUNK_BYTES = 2 << 30   # fp64 working set of the bound's reference per chunk of output columns


def _C():
    return _ext.load(True)


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _scale(x):
    return torch.tensor([x], device="cuda", dtype=torch.float32)


def _deq(sa, sb):
    """fp32(scale_a * scale_b), the kernel's dequantisation factor, as a Python float."""
    return (sa.double() * sb.double()).float().item()


def _full_mantissa(e, seed):
    """A positive fp32 in [2^e, 2^(e+1)) whose 24-bit significand has its lowest bit set."""
    m = int(torch.randint(0, 1 << 22, (1,), generator=torch.Generator().manual_seed(seed))) * 2 + 1
    return float((1 << 23) + m) * 2.0 ** (e - 23)


def _finite_codes(fmt):
    codes = torch.arange(256, dtype=torch.uint8)
    return codes[torch.isfinite(codes.view(fmt).float())].cuda()


def _random_codes(shape, fmt, seed, nonzero=False):
    """Uniform over every finite code of ``fmt`` (subnormals, +-0 and +-FP8_MAX included)."""
    codes = _finite_codes(fmt)
    if nonzero:
        codes = codes[codes.view(fmt).float() != 0]
    return codes[torch.randint(len(codes), shape, device="cuda", generator=_gen(seed))].view(fmt)


def _poisoned8(t, ld=None):
    """``t`` (fp8 [rows, K]) as a view into a buffer of POISON bytes with two extra rows before and after; the row
    stride ``ld`` is a multiple of 16 above K (default: 16 bytes before the view and at least 16 after), and the view
    starts 16-byte aligned."""
    rows, K = t.shape
    col0 = 16 if ld is None else 0
    ld = -(-K // 16) * 16 + 32 if ld is None else ld
    assert ld % 16 == 0 and ld > K + col0 - 1
    buf = torch.full((rows + 4, ld), POISON, device="cuda", dtype=torch.uint8)
    view = buf[2:2 + rows, col0:col0 + K]
    view.copy_(t.view(torch.uint8))
    return view.view(t.dtype)


def _same_bits(tag, got, want):
    """Bit-identical bf16, except that a NaN may carry any sign and payload."""
    gn, wn = torch.isnan(got.float()), torch.isnan(want.float())
    bad = (got.view(torch.int16) != want.view(torch.int16)) & ~(gn & wn)
    if bad.any():
        idx = bad.nonzero()[:4].tolist()
        ex = ", ".join(f"{tuple(i)}: got {got[tuple(i)].item():.6g} want {want[tuple(i)].item():.6g}" for i in idx)
        raise AssertionError(f"{tag}: {int(bad.sum())} of {bad.numel()} elements differ; {ex}")


def _exact_sum(p, c):
    """p + c in fp64, asserting it is exact (TwoSum's error term is zero): the test's premise, not the kernel's."""
    s = p + c
    bp = s - c
    err = (p - bp) + (c - (s - bp))
    assert bool((err == 0).all()), "the expected value is not exact in fp64"
    return s


def _expected(acc, deq, c=None):
    """bf16(fp32(acc * deq (+ c))) from the exact fp64 accumulator; acc * deq is exact in fp64 for every design here
    (at most 32 significant bits times 24), and so is the sum with c (asserted).  A zero sum is +0, as the
    accumulator, which starts at +0, makes of -0 products."""
    p = acc * deq + 0.0
    if c is not None:
        p = _exact_sum(p, c.double())
    return p.float().to(BF16)


def _gemm(a8, b8, out, sa, sb, accumulate=False, variant=1, bias=None):
    _C().gemm_fp8(a8, b8, out, sa, sb, accumulate, variant, bias)
    return out


def _on_grid(shape, deq, seed):
    """bf16 values deq * n, n an integer in [-512, 512]: with an integer accumulator of at most 2^10, acc * deq + c
    spans at most 36 bits, so it is exact in fp64."""
    n = torch.randint(-512, 513, shape, device="cuda", generator=_gen(seed)).double()
    return (n * deq).to(BF16)


# ------------------------------------------------------------------------------------------------------------------
# a. exact designs
# ------------------------------------------------------------------------------------------------------------------
# one K step, one 16-byte TMA row, ragged tails either side of one and of four 128-element K blocks, a long ragged K,
# and 128 K blocks (the 4-stage ring wraps 32 times)
ONE_TERM_K = [1, 16, 33, 127, 128, 129, 512 + 16, 16384]


@pytest.mark.parametrize("variant", [1, 2])
@pytest.mark.parametrize("a_fmt", list(FMTS))
@pytest.mark.parametrize("K", ONE_TERM_K)
def test_one_term_per_output(K, a_fmt, variant):
    """Row i of A has one nonzero, at k_i; the k_i run over every K position.  Every output is one product of two
    fp8 values, exact in fp32 whatever the accumulation precision, so every element is pinned bit for bit at every
    value B takes (all finite e4m3 codes, subnormals included)."""
    fmt = FMTS[a_fmt]
    M, N = max(K, 300), 272
    k_of_row = torch.randperm(K, device="cuda", generator=_gen(K))[torch.arange(M, device="cuda") % K]
    a_val = _random_codes((M,), fmt, seed=K + 1, nonzero=True)
    a8 = torch.zeros(M, K, device="cuda", dtype=torch.uint8)
    a8[torch.arange(M, device="cuda"), k_of_row] = a_val.view(torch.uint8)
    a8 = a8.view(fmt)
    b8 = _random_codes((N, K), E4M3, seed=K + 2)
    sa, sb = _scale(_full_mantissa(0, 1)), _scale(_full_mantissa(-3, 2))
    acc = a_val.double()[:, None] * b8.double()[:, k_of_row].t()
    want = _expected(acc, _deq(sa, sb))
    buf, view = _out_view(M, N, float("nan"))
    before = buf.clone()
    _gemm(_poisoned8(a8), _poisoned8(b8), view, sa, sb, variant=variant)
    tag = f"K{K} {a_fmt} v{variant}"
    assert _outside_unchanged(buf, before, M, N), f"{tag}: wrote outside the output view"
    _same_bits(tag, view, want)


def _sparse_ints(M, N, K, a_fmt, seed):
    """(a8, b8, exact fp64 A @ B^T): every row of A has nnz nonzeros at distinct K positions taken in turn from one
    permutation of K, with nnz large enough that every K position is used; B is dense in [-4, 4].  The nonzeros of A
    lie in [-4, 4] when nnz <= 64 and are +-1 up to nnz = 256, so sum_k |a_k b_k| <= 2^10 for every output."""
    g = _gen(seed)
    nnz = max(min(32, K), -(-K // M))
    assert nnz <= 256
    perm = torch.randperm(K, device="cuda", generator=g)
    pos = perm[(torch.arange(M, device="cuda")[:, None] * nnz + torch.arange(nnz, device="cuda")) % K]
    vals = torch.randint(1, 5 if nnz <= 64 else 2, (M, nnz), device="cuda", generator=g).float()
    vals *= torch.randint(0, 2, (M, nnz), device="cuda", generator=g).float() * 2 - 1
    A = torch.zeros(M, K, device="cuda").scatter_(1, pos, vals)
    B = torch.randint(-4, 5, (N, K), device="cuda", generator=g).float()
    exact = A.double() @ B.double().t()
    return A.to(FMTS[a_fmt]), B.to(E4M3), exact


def _modes(M, N, K, a_fmt, variant, seed, sa, sb, poison=False):
    """Run overwrite, accumulate and (e4m3 A) bias mode on one sparse-integer problem and compare bit for bit."""
    a8, b8, acc = _sparse_ints(M, N, K, a_fmt, seed)
    deq = _deq(sa, sb)
    if poison:
        a8, b8 = _poisoned8(a8), _poisoned8(b8)
    tag = f"M{M} N{N} K{K} {a_fmt} v{variant} deq {deq:.9g}"
    buf, view = _out_view(M, N, float("nan"))
    before = buf.clone()
    _gemm(a8, b8, view, sa, sb, variant=variant)
    assert _outside_unchanged(buf, before, M, N), f"{tag}: overwrite wrote outside its view"
    _same_bits(tag, view, _expected(acc, deq))
    c_old = _on_grid((M, N), deq, seed + 1)
    buf, view = _out_view(M, N, c_old)
    before = buf.clone()
    _gemm(a8, b8, view, sa, sb, accumulate=True, variant=variant)
    assert _outside_unchanged(buf, before, M, N), f"{tag}: accumulate wrote outside its view"
    _same_bits(tag + " acc", view, _expected(acc, deq, c_old))
    if a_fmt == "e4m3":
        bias = _on_grid((N,), deq, seed + 2)
        buf, view = _out_view(M, N, float("nan"))
        _gemm(a8, b8, view, sa, sb, variant=variant, bias=bias)
        _same_bits(tag + " bias", view, _expected(acc, deq, bias.expand(M, N)))


SPARSE_SHAPES = {**{k: (M, N, K, "e5m2" if f == E5M2 else "e4m3") for k, (M, N, K, f) in GEMM_SHAPES.items()},
                 "many-tiles-per-cta": (6144, 5120, 512, "e4m3")}


@pytest.mark.parametrize("variant", [1, 2])
@pytest.mark.parametrize("case", list(SPARSE_SHAPES))
def test_sparse_integer_sums(case, variant):
    M, N, K, a_fmt = SPARSE_SHAPES[case]
    _modes(M, N, K, a_fmt, variant, seed=40, sa=_scale(_full_mantissa(-2, 3)), sb=_scale(_full_mantissa(-6, 4)))
    torch.cuda.empty_cache()


@pytest.mark.parametrize("variant", [1, 2])
@pytest.mark.parametrize("a_fmt", list(FMTS))
def test_every_code_pair(a_fmt, variant):
    """K = 1: A runs over all 256 codes of its format, B over all 256 e4m3 codes.  NaN codes give NaN rows and columns,
    e5m2 +-Inf times a nonzero code +-Inf and times zero NaN; every finite pair, subnormals included, is exact."""
    fmt = FMTS[a_fmt]
    codes = torch.arange(256, device="cuda", dtype=torch.uint8)[:, None]
    a8, b8 = _poisoned8(codes.view(fmt), ld=16), _poisoned8(codes.view(E4M3), ld=16)
    one = _scale(1.0)
    out = torch.full((256, 256), float("nan"), device="cuda", dtype=BF16)
    _gemm(a8, b8, out, one, one, variant=variant)
    want = _expected(codes.view(fmt).double() * codes.view(E4M3).double().t(), 1.0)
    # a flushing tensor core would show here first: count the pairs with a subnormal operand that differ
    finite = torch.isfinite(want.float())
    with_sub = (_subnormal(codes.view(fmt)) | _subnormal(codes.view(E4M3)).t()) & finite
    diff = (out.view(torch.int16) != want.view(torch.int16)) & finite
    print(f"\n{a_fmt} x e4m3 v{variant}: {int(diff.sum())} finite pairs differ, {int((diff & with_sub).sum())} of the "
          f"{int(with_sub.sum())} pairs with a subnormal operand")
    _same_bits(f"{a_fmt} x e4m3 v{variant}", out, want)


def _subnormal(t):
    v = t.float().abs()
    return (v < torch.finfo(t.dtype).smallest_normal) & (v != 0)


# scale exponents from 2^-30 to 2^20, each with a full 24-bit significand
SCALE_EXPONENTS = [(-30, 20), (20, -30), (-30, -10), (20, 0), (-7, 5), (0, 0), (-1, -1)]


@pytest.mark.parametrize("variant", [1, 2])
def test_scales_with_full_mantissas(variant):
    """deq = fp32(scale_a * scale_b) exactly as the contract has it: a scale dropped, used twice or inverted, or a
    product rounded differently, changes elements."""
    for i, (ea, eb) in enumerate(SCALE_EXPONENTS):
        sa, sb = _scale(_full_mantissa(ea, 10 + i)), _scale(_full_mantissa(eb, 20 + i))
        _modes(300, 528, 160, "e4m3" if i % 2 else "e5m2", variant, seed=50 + i, sa=sa, sb=sb)


EDGE_M = [1, 63, 64, 65, 127, 128, 129, 255, 256, 257, 300]
EDGE_N = [16, 240, 256, 272, 528]
# M, N and K crossed sparsely: every value of each, each K with two different (M, N)
EDGE_SHAPES = [(EDGE_M[i % 11], EDGE_N[(3 * i) % 5], ONE_TERM_K[i % 8], "e5m2" if i % 3 == 1 else "e4m3")
               for i in range(16)]


@pytest.mark.parametrize("variant", [1, 2])
@pytest.mark.parametrize("M,N,K,a_fmt", EDGE_SHAPES)
def test_edge_shapes(M, N, K, a_fmt, variant):
    _modes(M, N, K, a_fmt, variant, seed=M + N + K, sa=_scale(_full_mantissa(3, M)), sb=_scale(_full_mantissa(-9, N)),
           poison=True)


@pytest.mark.parametrize("M,N,K", [(129, 272, 129), (300, 528, 16384)])
def test_edge_shapes_auto_variant(M, N, K):
    _modes(M, N, K, "e4m3", 3, seed=7, sa=_scale(_full_mantissa(1, 5)), sb=_scale(_full_mantissa(-4, 6)), poison=True)


# ------------------------------------------------------------------------------------------------------------------
# b. random data at the training shapes: every element against the truncation bound
# ------------------------------------------------------------------------------------------------------------------
def _bound_chunks(a8, b8, deq):
    """Per chunk of output columns: (j0, j1, exact unscaled sum, 2^-13 deq sum_t (|S_(t-1)| + sum_(k in t)|a_k b_k|)),
    all in fp64, the sums taken one k32 slice at a time in ascending K."""
    M, K = a8.shape
    N = b8.shape[0]
    A = a8.double()
    Aa = A.abs()
    cols = max(256, CHUNK_BYTES // (24 * M) // 256 * 256)
    for j0 in range(0, N, cols):
        j1 = min(N, j0 + cols)
        B = b8[j0:j1].double()
        S = torch.zeros(M, j1 - j0, device="cuda", dtype=torch.float64)
        E = torch.zeros_like(S)
        for k0 in range(0, K, 32):
            k1 = min(K, k0 + 32)
            E.add_(S.abs())
            E.addmm_(Aa[:, k0:k1], B[:, k0:k1].abs().t())
            S.addmm_(A[:, k0:k1], B[:, k0:k1].t())
        yield j0, j1, S, E.mul_(2.0 ** -13 * deq)
        del S, E, B


def _ratio(got, exact, bound):
    """The least c each element needs: (|got - exact| - 2^-8 |exact|) / bound; NaN / Inf outputs need c = inf."""
    excess = (got.double() - exact).abs_().sub_(exact.abs().mul_(2.0 ** -8))
    r = torch.where(excess <= 0, torch.zeros_like(excess), excess / bound)
    return torch.where(torch.isnan(r), torch.full_like(r, float("inf")), r)


def _worst_c(a8, b8, deq, outs):
    """outs: {name: (got, C_old or None)} -> {name: the largest c any element needs}."""
    worst = {name: 0.0 for name in outs}
    for j0, j1, S, bound in _bound_chunks(a8, b8, deq):
        exact0 = S.mul_(deq)
        for name, (got, old) in outs.items():
            exact = exact0 if old is None else exact0 + old[:, j0:j1].double()
            worst[name] = max(worst[name], _ratio(got[:, j0:j1], exact, bound).max().item())
    return worst


@pytest.mark.parametrize("case", list(GEMM_SHAPES))
def test_random_data_elementwise_bound(case):
    M, N, K, a_fmt = GEMM_SHAPES[case]
    a8, sa, b8, sb = _operands(M, N, K, a_fmt)
    deq = _deq(sa, sb)
    outs = {}
    for v in (1, 2):
        out = torch.empty(M, N, device="cuda", dtype=BF16)
        outs[f"v{v}"] = (_gemm(a8, b8, out, sa, sb, variant=v), None)
    std = outs["v1"][0].float().std().item()
    old = (std * torch.randn(M, N, device="cuda", generator=_gen(8))).to(BF16)
    for v in (1, 2):
        outs[f"v{v} acc"] = (_gemm(a8, b8, old.clone(), sa, sb, accumulate=True, variant=v), old)
    worst = _worst_c(a8, b8, deq, outs)
    print(f"\n{case}: element c " + "  ".join(f"{n} {c:.3g}" for n, c in worst.items()))
    for name, c in worst.items():
        assert c <= ELEM_C, f"{case} {name}: an element needs c = {c:.3g} > {ELEM_C}"
    del outs, old
    torch.cuda.empty_cache()


def test_bound_rejects_small_errors():
    """The bound is not vacuous: one element off by 1 %, or one row off by 2 bf16 ulps, fails it."""
    M, N, K, a_fmt = GEMM_SHAPES["odd-e4m3"]
    a8, sa, b8, sb = _operands(M, N, K, a_fmt)
    deq = _deq(sa, sb)
    out = _gemm(a8, b8, torch.empty(M, N, device="cuda", dtype=BF16), sa, sb)
    (_, _, S, bound), = list(_bound_chunks(a8, b8, deq))
    exact = S.mul_(deq)
    assert _ratio(out, exact, bound).max().item() <= ELEM_C
    i, j = divmod(int((exact.abs() / bound).argmax()), N)      # the element where the bound is tightest
    one = out.clone()
    one[i, j] = (out[i, j].float() * 1.01).to(BF16)
    c_one = _ratio(one, exact, bound).max().item()
    row = out.clone()
    row[M - 1] = (row[M - 1].view(torch.int16) + 2).view(BF16)
    c_row = _ratio(row, exact, bound).max().item()
    print(f"\nperturbed: one element by 1 % needs c = {c_one:.3g}, the last row by 2 ulps c = {c_row:.3g}")
    assert c_one > ELEM_C and c_row > ELEM_C


# ------------------------------------------------------------------------------------------------------------------
# c. position independence
# ------------------------------------------------------------------------------------------------------------------
# (r0, r1, c0, c1): windows across the 64-, 128- and 256-row and the 256-column boundaries
WINDOWS = [(60, 70, 240, 272), (120, 140, 496, 528), (250, 262, 16, 784), (100, 400, 240, 528), (255, 257, 0, 16),
           (0, 600, 256, 512)]


@pytest.mark.parametrize("a_fmt", list(FMTS))
def test_bits_do_not_depend_on_position(a_fmt):
    M, N, K = 600, 800, 4096
    a8, sa, b8, sb = _operands(M, N, K, FMTS[a_fmt], seed=60)
    full = {v: _gemm(a8, b8, torch.empty(M, N, device="cuda", dtype=BF16), sa, sb, variant=v) for v in (1, 2, 3)}
    for v in (2, 3):
        _same_bits(f"{a_fmt} variant {v} vs 1", full[v], full[1])
    _same_bits(f"{a_fmt} second call", _gemm(a8, b8, torch.empty_like(full[1]), sa, sb), full[1])
    buf, view = _out_view(M, N, float("nan"))
    _same_bits(f"{a_fmt} into a view", _gemm(a8, b8, view, sa, sb), full[1])
    for r0, r1, c0, c1 in WINDOWS:
        for v in (1, 2, 3):
            sub = _gemm(a8[r0:r1], b8[c0:c1], torch.empty(r1 - r0, c1 - c0, device="cuda", dtype=BF16), sa, sb,
                        variant=v)
            _same_bits(f"{a_fmt} rows {r0}:{r1} cols {c0}:{c1} v{v}", sub, full[1][r0:r1, c0:c1])


# ------------------------------------------------------------------------------------------------------------------
# d. non-finite operands, empty sizes, operands cast with a tiny amax
# ------------------------------------------------------------------------------------------------------------------
NAN_AT = [(0, 0, 0), (299, 527, 319), (129, 257, 128), (255, 263, 31)]   # (i, j, k)


@pytest.mark.parametrize("variant", [1, 2])
def test_nonfinite_operands(variant):
    M, N, K = 300, 528, 320
    for i, j, k in NAN_AT:
        a8, sa, b8, sb = _operands(M, N, K, E4M3, seed=70)
        a8.view(torch.uint8)[i, k] = POISON
        out = _gemm(a8, b8, torch.empty(M, N, device="cuda", dtype=BF16), sa, sb, variant=variant)
        rows = torch.zeros(M, N, dtype=torch.bool, device="cuda")
        rows[i] = True
        assert torch.equal(torch.isnan(out), rows), f"NaN at A[{i},{k}] v{variant}: not exactly row {i} is NaN"
        a8, sa, b8, sb = _operands(M, N, K, E4M3, seed=70)
        b8.view(torch.uint8)[j, k] = POISON
        out = _gemm(a8, b8, out, sa, sb, variant=variant)
        cols = torch.zeros(M, N, dtype=torch.bool, device="cuda")
        cols[:, j] = True
        assert torch.equal(torch.isnan(out), cols), f"NaN at B[{j},{k}] v{variant}: not exactly column {j} is NaN"
        for inf_code in (0x7C, 0xFC):   # e5m2 +Inf, -Inf
            a8, sa, b8, sb = _operands(M, N, K, E5M2, seed=71)
            a8.view(torch.uint8)[i, k] = inf_code
            b8.view(torch.uint8)[j, k] = 0x00
            b8.view(torch.uint8)[(j + 1) % N, k] = 0x80   # -0
            out = _gemm(a8, b8, out, sa, sb, variant=variant)
            want = (a8[i].double() * b8.double()).sum(1) * _deq(sa, sb)   # Inf arithmetic, NaN where b[:, k] is 0
            tag = f"Inf {inf_code:#x} at A[{i},{k}] v{variant}"
            _same_bits(tag, out[i:i + 1], want.float().to(BF16)[None])
            others = torch.ones(M, dtype=torch.bool, device="cuda")
            others[i] = False
            assert bool(torch.isfinite(out[others]).all()), f"{tag}: another row is not finite"


@pytest.mark.parametrize("variant", [1, 2, 3])
def test_k0_m0_n0(variant):
    """K = 0: overwrite writes zeros, accumulate leaves the view bit-identical.  M = 0 or N = 0: no launch, no
    error."""
    M, N = 129, 272
    one = _scale(1.0)
    for a_fmt, fmt in FMTS.items():
        a8 = torch.zeros(M, 16, device="cuda", dtype=fmt)[:, :0]
        b8 = torch.zeros(N, 16, device="cuda", dtype=E4M3)[:, :0]
        for acc in (False, True):
            buf, view = _out_view(M, N, _on_grid((M, N), 1.0, 80))
            before = buf.clone()
            _gemm(a8, b8, view, one, one, accumulate=acc, variant=variant)
            assert _outside_unchanged(buf, before, M, N)
            want = before[2:2 + M, 8:8 + N] if acc else torch.zeros(M, N, device="cuda", dtype=BF16)
            _same_bits(f"K0 {a_fmt} acc={acc}", view, want)
        a8 = torch.zeros(M, 64, device="cuda", dtype=fmt)
        b8 = torch.zeros(N, 64, device="cuda", dtype=E4M3)
        torch.cuda.synchronize()
        n0 = _ext.launch_count()
        for acc in (False, True):
            _gemm(a8[:0], b8, torch.empty(0, N, device="cuda", dtype=BF16), one, one, accumulate=acc, variant=variant)
            _gemm(a8, b8[:0], torch.empty(M, 0, device="cuda", dtype=BF16), one, one, accumulate=acc, variant=variant)
        torch.cuda.synchronize()
        assert _ext.launch_count() == n0, "an empty GEMM launched a kernel"


def test_tiny_amax_operands_give_finite_products():
    """Operands cast with the clamped scale (amax below FP8_MAX / FLT_MAX): the product only has to be finite, since
    deq falls below fp32's normal range."""
    g = _gen(90)
    x = (1e-37 * torch.randn(256, 512, device="cuda", generator=g)).to(BF16)
    x[:, ::3] = 0
    w = (0.02 * torch.randn(528, 512, device="cuda", generator=g)).to(BF16)
    x8, _, sx = _C().fp8_cast_transpose(x, _C().fp8_amax(x), False, True, False)
    w8, _, sw = _C().fp8_cast_transpose(w, _C().fp8_amax(w), False, True, False)
    assert sx.item() == 2.0 ** -128
    for v in (1, 2):
        out = _gemm(x8, w8, torch.empty(256, 528, device="cuda", dtype=BF16), sx, sw, variant=v)
        assert bool(torch.isfinite(out).all()), f"v{v}: {int((~torch.isfinite(out)).sum())} non-finite outputs"


# ------------------------------------------------------------------------------------------------------------------
# e. refusals before any launch
# ------------------------------------------------------------------------------------------------------------------
def test_gemm_fp8_refusals():
    M, N, K = 256, 272, 128
    C = _C()
    a8 = torch.zeros(M, K + 16, device="cuda", dtype=E4M3)
    a5 = torch.zeros(M, K, device="cuda", dtype=E5M2)
    b8 = torch.zeros(N, K + 16, device="cuda", dtype=E4M3)
    out = torch.empty(M, N + 16, device="cuda", dtype=BF16)
    one = _scale(1.0)
    A, B, O = a8[:, :K], b8[:, :K], out[:, :N]
    bias = torch.zeros(N, device="cuda", dtype=BF16)
    cases = [
        (lambda: C.gemm_fp8(A.to(BF16), B, O, one, one), "a must be float8"),
        (lambda: C.gemm_fp8(A, B.float().to(BF16), O, one, one), "b must be float8"),
        (lambda: C.gemm_fp8(A, B.float().to(E5M2), O, one, one), "b must be float8_e4m3fn"),
        (lambda: C.gemm_fp8(A, B, O.float(), one, one), "out must be bfloat16"),
        (lambda: C.gemm_fp8(A, B, out[:, :N - 16], one, one), "wrong shape"),
        (lambda: C.gemm_fp8(A, B, torch.empty(N, M, device="cuda", dtype=BF16).t(), one, one), "contiguous last"),
        (lambda: C.gemm_fp8(torch.zeros(M, K + 8, device="cuda", dtype=E4M3)[:, :K], B, O, one, one),
         "multiples of 16"),
        (lambda: C.gemm_fp8(A, torch.zeros(N, K + 8, device="cuda", dtype=E4M3)[:, :K], O, one, one),
         "multiples of 16"),
        (lambda: C.gemm_fp8(A, B, torch.empty(M, N + 8, device="cuda", dtype=BF16)[:, :N], one, one),
         "multiples of 16"),
        (lambda: C.gemm_fp8(a8[:, 8:8 + K], B, O, one, one), "A must start"),
        (lambda: C.gemm_fp8(A, b8[:, 8:8 + K], O, one, one), "B must start"),
        (lambda: C.gemm_fp8(A, B, out[:, 4:4 + N], one, one), "C must start"),
        (lambda: C.gemm_fp8(A, b8[:, :K - 16], O, one, one), "inner dimensions differ"),
        (lambda: C.gemm_fp8(A, B, O, one.cpu(), one), "scale_a must be"),
        (lambda: C.gemm_fp8(A, B, O, one, one.double()), "scale_b must be"),
        (lambda: C.gemm_fp8(A, B, O, torch.ones(2, device="cuda"), one), "scale_a must be"),
        (lambda: C.gemm_fp8(a5, B, O, one, one, False, 0, bias), "bias needs a float8_e4m3fn"),
        (lambda: C.gemm_fp8(A, B, O, one, one, True, 0, bias), "bias cannot be combined with accumulate"),
        (lambda: C.gemm_fp8(a8[:, :0], b8[:, :0], O, one, one, False, 0, bias), "bias needs K >= 1"),
    ]
    for i, (call, match) in enumerate(cases):
        _refused(call, match)


def test_cast_refusals():
    C = _C()
    x = torch.randn(64, 128, device="cuda").to(BF16)
    amax = C.fp8_amax(x)
    cases = [
        (lambda: C.fp8_cast_transpose(x, amax.double(), False), "amax must be"),
        (lambda: C.fp8_cast_transpose(x, amax.expand(2).contiguous(), False), "amax must be"),
        (lambda: C.fp8_cast_transpose(x, amax.cpu(), False), "amax must be"),
        (lambda: C.fp8_cast_transpose(x[:0], amax, False), "empty"),
        (lambda: C.fp8_cast_transpose(x, amax, True, False, False), "at least one layout"),
        (lambda: C.fp8_cast_transpose(x.float(), amax, False), "x must be bfloat16"),
    ]
    for call, match in cases:
        _refused(call, match)


# ------------------------------------------------------------------------------------------------------------------
# the casts over the whole bf16 range
# ------------------------------------------------------------------------------------------------------------------
def _all_finite_bf16():
    """Every finite bf16 value, both signs, as fp32 on the device."""
    pos = torch.arange(0, 0x7F80, device="cuda", dtype=torch.int32).to(torch.int16).view(BF16).float()
    return torch.cat([pos, -pos[1:]])


def _amax_per_binade():
    """One amax in every bf16 binade, from the least subnormal (2^-133) to bf16's largest finite value, each with a
    different significand, plus both ends exactly."""
    vals = [2.0 ** -133, torch.finfo(BF16).max]
    for e in range(-133, 128):
        m = (37 * (e + 133)) % 128 if e >= -126 else 0          # subnormal binades: the power of two itself
        vals.append((1 + m / 128) * 2.0 ** e)
    return torch.tensor(vals, dtype=torch.float32).to(BF16).float().unique()


@pytest.mark.parametrize("fmt", list(FMTS))
def test_cast_whole_range(fmt):
    """Every finite bf16 x with |x| <= amax, at an amax in every binade: bit for bit against the reference
    quantisation, no NaN, ``|q - x scale| <= u |x scale| + (half the least subnormal) + 2^-24 |x scale|`` in fp64 and
    ``|q| <= FP8_MAX``."""
    dtype = FMTS[fmt]
    fmax = torch.finfo(dtype).max
    u, half_sub = (2.0 ** -4, 2.0 ** -10) if dtype == E4M3 else (2.0 ** -3, 2.0 ** -17)
    xs = _all_finite_bf16()
    for amax_v in _amax_per_binade().tolist():
        x = xs[xs.abs() <= amax_v]
        n = x.numel()
        x = torch.nn.functional.pad(x, (0, -n % 256)).view(-1, 256).to(BF16)
        amax = _scale(amax_v)
        x8, _, si = _C().fp8_cast_transpose(x, amax, dtype == E5M2, True, False)
        want8, want_si = ref.fp8_quantize(x.cpu(), dtype, amax=amax.cpu())
        tag = f"{fmt} amax {amax_v:.6g}"
        assert torch.equal(x8.view(torch.uint8).cpu(), want8.view(torch.uint8)), f"{tag}: differs from the reference"
        assert torch.equal(si.cpu(), want_si), f"{tag}: scale_inv {si.item()} vs {want_si.item()}"
        q = x8.double()
        assert not bool(torch.isnan(q).any()), f"{tag}: a finite input quantised to NaN"
        assert q.abs().max().item() <= fmax, tag
        scale = min(fmax / amax_v, torch.finfo(torch.float32).max)
        scale = torch.tensor(scale, dtype=torch.float32).double().item()   # the fp32 scale, correctly rounded
        xsd = x.double() * scale
        err = (q - xsd).abs()
        ok = err <= (u + 2.0 ** -24) * xsd.abs() + half_sub
        assert bool(ok.all()), f"{tag}: {int((~ok).sum())} elements outside the rounding bound"
