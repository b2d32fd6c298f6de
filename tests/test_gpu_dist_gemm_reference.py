"""The tensor-parallel modes of the wgmma GEMM and the partial-sum reduce, on one GPU, against the plain GEMM
bit for bit and against fp64.

Ranks are emulated as in ``test_gpu_vocab_reference.py``: every rank's buffer is a separate tensor on the same device,
their ``data_ptr()`` values form the peer-pointer lists, and the ranks' calls run in rank order on one stream.  Signal
pads are plain int32 tensors of ``SYMM_MAX_CHANNELS x 8``.  One GPU cannot test memory ordering across GPUs; the
``multigpu`` tests stay the check over real NVLink.

Contracts (the launcher comment in ``gemm_wgmma.cu``):
- ``gemm_ag`` (all-gather by communication CTAs, then the GEMM) and ``gemm_dist`` modes 1 and 2 keep the plain GEMM's
  K order, so they are bit-identical to ``gemm(..., variant=2)`` on the assembled operands, with the same bias or
  accumulate.
- ``gemm_dist`` modes 3 and 4 start every tile at this rank's K slice.  They must be within the fp64 element bound of
  ``test_gpu_gemm_reference.py`` (``2^-8 |exact| + ELEM_C K 2^-24 (|A| @ |B|)``), and bit-identical where the rotation
  is 0.
- ``tp_reduce_parts`` is bit-identical to an fp32 sum of the parts in part order, then the residual, then one bf16
  rounding.  Against fp64 the reduced rows must be within (1 + 2^-8) x (2^-8 |exact| + the partials' GEMM element
  bounds + t 2^-24 sum |terms|): the final rounding, each pushed partial's rounding and accumulation, and the fp32 sum
  of t + 1 terms.  The rows must also be within 2^-8 |S| + t 2^-24 sum |terms| of the fp64 sum S of the partials the
  GEMMs actually pushed: that half sees a 2-ulp error in one element.

Every operand sits where a wrong read or write shows: a peer's rows or bytes outside its owner's slice are NaN at the
call, staging slots and outputs are views inside allocations whose outside bits must not change, and an overwritten
output starts out NaN.

The kernels spin on flags and pads, and trap after 8 s.  No test here can reach that: before each launch the test
asserts that every emulated peer's arrival is already in ``pads[rank]``, and the only flags the kernel waits on are
the ones its own communication CTAs set.
"""
import pytest
import torch

from distributed_training_guide_b200 import _ext
from test_gpu_gemm_reference import ELEM_C, _evaluate
from test_gpu_kernels_reference import _refused

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16
NAN = float("nan")
PAD = 64            # sentinel elements before and after every guarded view (128 bytes keep 16-byte alignment)
U = 2.0 ** -24


def _C():
    return _ext.load(True)


def _channels():
    return int(_C().SYMM_MAX_CHANNELS)


def _bits(t):
    return t.contiguous().view(torch.int16 if t.element_size() == 2 else torch.int32)


def _same(a, b):
    return torch.equal(_bits(a), _bits(b))


def _randn(shape, seed, std=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (std * torch.randn(*shape, device="cuda", generator=g)).to(BF16)


class _Guarded:
    """An n-element view inside an allocation with PAD elements of random bits before and after it."""

    def __init__(self, n, dtype=BF16, fill=NAN, seed=99):
        g = torch.Generator(device="cuda").manual_seed(seed)
        if dtype == BF16:
            self.buf = torch.randint(-2 ** 15, 2 ** 15, (n + 2 * PAD,), device="cuda", generator=g,
                                     dtype=torch.int32).to(torch.int16).view(BF16)
        else:
            self.buf = torch.randint(-2 ** 31, 2 ** 31 - 1, (n + 2 * PAD,), device="cuda", generator=g, dtype=dtype)
        self.n = n
        self.view = self.buf[PAD:PAD + n]
        if fill is not None:
            self.view.fill_(fill)
        self._edges = self.edges().clone()

    def edges(self):
        return torch.cat([_bits(self.buf[:PAD]), _bits(self.buf[PAD + self.n:])])

    def intact(self):
        return torch.equal(self.edges(), self._edges)


def _out(M, N, fill=NAN):
    """An [M, N] output view (row stride N + 16) inside a guarded allocation; returns (guard, view)."""
    ld = N + 16
    g = _Guarded(M * ld, fill=None)
    v = g.view.view(M, ld)[:, 8:8 + N]
    if isinstance(fill, torch.Tensor):
        v.copy_(fill)
    else:
        v.fill_(fill)
    g._rest = v, _bits(g.view.view(M, ld)).clone()
    return g, v


def _out_intact(g):
    """Nothing outside the [M, N] view and outside the allocation's view changed."""
    v, before = g._rest
    now = _bits(g.view.view(before.shape))
    mask = torch.ones_like(now, dtype=torch.bool)
    mask[:, 8:8 + v.shape[1]] = False
    return g.intact() and torch.equal(now[mask], before[mask])


def _plain(A, B, b_kmajor, bias=None, old=None):
    """The plain CTA-pair GEMM A @ op(B) (+ bias, or + old in accumulate mode)."""
    out = old.clone() if old is not None else torch.empty(A.shape[0], B.shape[0] if b_kmajor else B.shape[1],
                                                          device="cuda", dtype=BF16)
    _C().gemm(A, B, out, False, b_kmajor, old is not None, 2, bias)
    return out


def _pads(t):
    return [torch.zeros(_channels() * 8, device="cuda", dtype=torch.int32) for _ in range(t)]


# ------------------------------------------------------------------------------------------------------------------
# gemm_ag: the all-gather of A's rows by communication CTAs inside the GEMM (A_MODE 3)
# ------------------------------------------------------------------------------------------------------------------
def _ag_run(t, r, rpp, K, N, n_comm, b_kmajor, with_bias, seed):
    C = _C()
    M = t * rpp
    lmt = rpp // 256
    W = _randn((N, K) if b_kmajor else (K, N), seed + 1, std=K ** -0.5)
    bias = _randn((N,), seed + 2) if with_bias else None
    bufs = [_Guarded(M * K, seed=seed + 10 + p) for p in range(t)]   # every row NaN, then the owner's slice
    pads = _pads(t)
    flags = _Guarded(M // 256, dtype=torch.int32, fill=None, seed=seed + 3)
    for call, (ag_epoch, bar_epoch) in enumerate([(5, 7), (6, 8)]):
        X = _randn((M, K), seed + 20 + call)
        for p in range(t):   # fresh rows in every peer; buffer r's other rows hold NaN (first call) or stale rows
            bufs[p].view.view(M, K)[p * rpp:(p + 1) * rpp].copy_(X[p * rpp:(p + 1) * rpp])
        flags.view.fill_(ag_epoch - 1)
        flags.view[r * lmt:(r + 1) * lmt] = ag_epoch - 3   # own tiles: never waited for, never written
        pads[r].fill_(bar_epoch)                       # every emulated peer has already arrived
        before = [_bits(b.view).clone() for b in bufs]
        pads_before = [p.clone() for p in pads]
        flags_before = flags.view.clone()
        og, out = _out(M, N)
        # the kernel waits only on pads[r] and on the flags of remote tiles, which its own communication CTAs set
        assert bool((pads[r] == bar_epoch).all())
        assert bool((flags.view < ag_epoch).all())
        C.gemm_ag([b.view.data_ptr() for b in bufs], W, out, b_kmajor, r, rpp, flags.view, ag_epoch,
                  [p.data_ptr() for p in pads], bar_epoch, n_comm, bias)
        torch.cuda.synchronize()
        tag = (f"t{t} r{r} rpp{rpp} K{K} N{N} n_comm{n_comm} {'fwd' if b_kmajor else 'dgrad'}"
               f"{' bias' if bias is not None else ''} call{call}")
        want = _plain(X, W, b_kmajor, bias)
        diff = int((_bits(out) != _bits(want)).sum())
        assert diff == 0, f"{tag}: {diff} of {M * N} elements differ from the plain GEMM"
        assert _out_intact(og), f"{tag}: wrote outside the output view"
        assert _same(bufs[r].view.view(M, K), X), f"{tag}: rank {r}'s buffer is not the gathered rows"
        for p in range(t):
            assert bufs[p].intact(), f"{tag}: wrote outside peer {p}'s buffer"
            if p != r:
                assert torch.equal(_bits(bufs[p].view), before[p]), f"{tag}: peer {p}'s buffer changed"
        remote = torch.ones(M // 256, dtype=torch.bool, device="cuda")
        remote[r * lmt:(r + 1) * lmt] = False
        assert bool((flags.view[remote] == ag_epoch).all()), f"{tag}: a remote tile's flag is not ag_epoch"
        assert torch.equal(flags.view[~remote], flags_before[~remote]), f"{tag}: an own tile's flag changed"
        assert flags.intact(), f"{tag}: wrote outside the flags"
        for p in range(t):
            want_pad = pads_before[p].clone().view(-1, 8)
            want_pad[:2 * n_comm, r] = bar_epoch
            assert torch.equal(pads[p], want_pad.view(-1)), f"{tag}: pad of rank {p}"


# (t, rpp, K, N, n_comm, b_kmajor, bias).  Remote tiles (t - 1) * rpp / 256 against 2 * n_comm copying CTAs: 7 over
# 2 and 4, 9 over 4, 3 over 8 (CTAs without a tile), 14 over 2.  N tails: 1376 = 11008 / 8 (down_proj's dgrad at
# TP 8), 16032 = 128256 / 8 (the lm_head at TP 8), 576 with a bias (Qwen2.5-7B's fused qkv at TP 8), 264 and 520.
AG_CASES = [
    (1, 256, 64, 264, 1, True, False),
    (1, 768, 4096, 576, 2, True, True),
    (2, 256, 64, 256, 1, True, True),
    (2, 512, 4096, 1376, 2, False, False),
    (2, 768, 8192, 520, 4, False, False),
    (4, 768, 2048, 576, 2, True, True),
    (4, 256, 3584, 576, 4, True, True),
    (4, 512, 5120, 1376, 1, False, False),
    (8, 256, 4096, 1376, 1, False, False),
    (8, 256, 4096, 16032, 4, True, False),
    (8, 512, 64, 264, 1, True, True),
    (8, 768, 1536, 520, 2, False, False),
]


@pytest.mark.parametrize("t,rpp,K,N,n_comm,b_kmajor,bias", AG_CASES)
def test_gemm_ag_matches_plain_gemm_bit_for_bit(t, rpp, K, N, n_comm, b_kmajor, bias):
    for r in sorted({0, t // 2, t - 1}):
        _ag_run(t, r, rpp, K, N, n_comm, b_kmajor, bias, seed=t * 100 + r + K + N)


REGISTRY_HIDDEN = [768, 896, 1536, 2048, 2560, 3072, 3584, 4096, 4608, 5120, 6144, 8192, 16384]


@pytest.mark.parametrize("K", REGISTRY_HIDDEN)
def test_gemm_ag_at_every_registry_hidden_size(K):
    """K is every hidden size the model registry trains (a copied tile is 256 K-element rows, in 32 KB pieces)."""
    _ag_run(4, 1, 256, K, 264, 2, True, True, seed=K)
    _ag_run(2, 1, 256, K, 256, 1, False, False, seed=K + 1)


# ------------------------------------------------------------------------------------------------------------------
# gemm_dist mode 2 (GEMM -> reduce-scatter push) and tp_reduce_parts
# ------------------------------------------------------------------------------------------------------------------
def _reduce_emulated(parts, res):
    acc = torch.zeros(parts.shape[1:], device="cuda", dtype=torch.float32)
    for p in range(parts.shape[0]):
        acc += parts[p].float()
    if res is not None:
        acc += res.float()
    return acc.to(BF16)


def _reduce_fracs(y, parts, res, exact, partial_bound):
    """Largest fraction of the two reduce bounds (module docstring) that any element of y uses: against the fp64 sum S
    of the pushed partials (plus residual), and against the exact result.  inf for a NaN."""
    t = parts.shape[0]
    pd = parts.double()
    terms = pd.abs().sum(0)
    S = pd.sum(0)
    if res is not None:
        terms += res.double().abs()
        S += res.double()
    yd = y.double()
    b_sum = 2.0 ** -8 * S.abs() + (1 + 2.0 ** -8) * t * U * terms
    b_exact = (1 + 2.0 ** -8) * (2.0 ** -8 * exact.abs() + partial_bound + t * U * terms)

    def worst(err, b):
        f = err / b.clamp_min(1e-300)
        f = torch.where(torch.isnan(f), torch.full_like(f, float("inf")), f)
        return f.max().item()
    return worst((yd - S).abs(), b_sum), worst((yd - exact).abs(), b_exact)


# (t, rpp, k, H, b_kmajor): k = 1376 (down_proj at TP 8: 1376 % 64 = 32), 16032 (the lm_head's dgrad at TP 8, B
# MN-major), 4000 (32000 / 8), 4096
RS_CASES = [
    (1, 256, 1376, 512, True),
    (2, 256, 1376, 520, True),
    (2, 512, 4096, 264, False),
    (4, 256, 4000, 512, True),
    (4, 256, 16032, 512, False),
    (8, 256, 1376, 512, True),
    (8, 256, 16032, 256, False),
    (8, 256, 4000, 264, False),
]


def _rs_run(t, rpp, k, H, b_kmajor, seed):
    """Every rank's GEMM pushes its partial into the t staging buffers; returns what the reduce tests need."""
    C = _C()
    T = t * rpp
    A = [_randn((T, k), seed + r) for r in range(t)]
    W = [_randn((H, k) if b_kmajor else (k, H), seed + 50 + r, std=k ** -0.5) for r in range(t)]
    stage = [_Guarded(t * rpp * H, seed=seed + 90 + p) for p in range(t)]
    full = []
    for r in range(t):
        C.gemm_dist(2, [A[r].data_ptr()], [W[r].data_ptr()], [s.view.data_ptr() + r * rpp * H * 2 for s in stage], T,
                    H, k, k, W[r].stride(0), H, b_kmajor, False, t, r, rpp)
        full.append(_plain(A[r], W[r], b_kmajor))
    torch.cuda.synchronize()
    return A, W, stage, full


@pytest.mark.parametrize("t,rpp,k,H,b_kmajor", RS_CASES)
def test_gemm_rs_push_and_reduce(t, rpp, k, H, b_kmajor):
    tag = f"t{t} rpp{rpp} k{k} H{H} {'nt' if b_kmajor else 'nn'}"
    A, W, stage, full = _rs_run(t, rpp, k, H, b_kmajor, seed=t + k + H)
    for p in range(t):
        assert stage[p].intact(), f"{tag}: wrote outside staging buffer {p}"
        sv = stage[p].view.view(t, rpp, H)
        for r in range(t):
            d = int((_bits(sv[r]) != _bits(full[r][p * rpp:(p + 1) * rpp])).sum())
            assert d == 0, f"{tag}: slot ({p}, {r}) differs from rows {p} of rank {r}'s plain GEMM in {d} elements"
    worst = [0.0, 0.0]
    for p in range(t):
        rows = slice(p * rpp, (p + 1) * rpp)
        exact = sum(A[r][rows].double() @ (W[r].double().t() if b_kmajor else W[r].double()) for r in range(t))
        partial_bound = sum(
            2.0 ** -8 * (A[r][rows].double() @ (W[r].double().t() if b_kmajor else W[r].double())).abs()
            + ELEM_C * k * U * (A[r][rows].double().abs() @ (W[r].double().t() if b_kmajor else W[r].double()).abs())
            for r in range(t))
        parts = stage[p].view.view(t, rpp, H)
        for with_res in (False, True):
            res_g = _Guarded(rpp * H, fill=None, seed=p + 7) if with_res else None
            res = res_g.view.view(rpp, H).copy_(_randn((rpp, H), seed=p + 8, std=4.0)) if with_res else None
            yg = _Guarded(rpp * H, seed=p + 9)
            y = yg.view.view(rpp, H)
            parts_before = _bits(parts).clone()
            _C().tp_reduce_parts(parts, res, y)
            torch.cuda.synchronize()
            sub = f"{tag} rank {p}{' + residual' if with_res else ''}"
            assert _same(y, _reduce_emulated(parts, res)), f"{sub}: not the fp32 sum in part order"
            assert yg.intact() and torch.equal(_bits(parts), parts_before), f"{sub}: wrote outside y"
            ex = exact + res.double() if with_res else exact
            f_sum, f_exact = _reduce_fracs(y, parts, res, ex, partial_bound)
            worst = [max(worst[0], f_sum), max(worst[1], f_exact)]
            assert f_sum <= 1 and f_exact <= 1, f"{sub}: bound fractions {f_sum:.3g} (sum) {f_exact:.3g} (exact)"
    print(f"\n{tag}: reduce bound used {worst[0]:.3f} (against the pushed partials), {worst[1]:.3f} (against fp64)")


def test_reduce_bound_rejects_wrong_slot_dropped_part_and_two_ulps():
    """The reduce bound is tight enough to see a partial pushed to the wrong owner, a dropped partial and a 2-ulp
    error in one element."""
    t, rpp, k, H = 4, 256, 1376, 512
    A, W, stage, full = _rs_run(t, rpp, k, H, True, seed=3)
    p = 1
    rows = slice(p * rpp, (p + 1) * rpp)
    exact = sum(A[r][rows].double() @ W[r].double().t() for r in range(t))
    pb = sum(2.0 ** -8 * (A[r][rows].double() @ W[r].double().t()).abs()
             + ELEM_C * k * U * (A[r][rows].double().abs() @ W[r].double().abs().t()) for r in range(t))
    parts = stage[p].view.view(t, rpp, H).clone()
    y = _reduce_emulated(parts, None)
    assert max(_reduce_fracs(y, parts, None, exact, pb)) <= 1
    wrong = parts.clone()
    wrong[2] = full[2][(p + 1) * rpp:(p + 2) * rpp]      # rank 2 pushed the next owner's rows into this slot
    assert max(_reduce_fracs(_reduce_emulated(wrong, None), wrong, None, exact, pb)) > 1, "wrong slot not rejected"
    dropped = parts[:t - 1]
    assert max(_reduce_fracs(_reduce_emulated(dropped, None), parts, None, exact, pb)) > 1, "dropped part not seen"
    i = int(y.float().abs().argmax())
    y2 = y.clone().view(-1)
    y2[i] = (y2[i:i + 1].view(torch.int16) + 2).view(BF16)[0]
    assert max(_reduce_fracs(y2.view(rpp, H), parts, None, exact, pb)) > 1, "2-ulp error not rejected"


# ------------------------------------------------------------------------------------------------------------------
# gemm_dist modes 1, 3 and 4
# ------------------------------------------------------------------------------------------------------------------
def _check_fp64(tag, A, B, got, old=None):
    c = _evaluate(A, B, {"kernel": got}, old)["kernel"][1]
    assert torch.isfinite(got).all(), f"{tag}: non-finite elements"
    assert c <= ELEM_C, f"{tag}: an element needs c = {c:.3g} > {ELEM_C}"
    return c


# (t, rpp) for mode 1 (rows of A per rank, multiples of 256) and modes 3 / 4 (K rows per rank, multiples of 64)
@pytest.mark.parametrize("t", [1, 2, 4, 8])
def test_gemm_dist_mode1_matches_plain_gemm(t):
    C = _C()
    rpp, K, N = 256, 1376, 520
    M = t * rpp
    for b_kmajor in (True, False):
        W = _randn((N, K) if b_kmajor else (K, N), t + 1, std=K ** -0.5)
        X = _randn((M, K), t + 2)
        # every rank's [rpp, K] slice, followed by NaN rows in the same allocation (a read past rpp rows shows)
        srcs = []
        for p in range(t):
            g = _Guarded((rpp + 8) * K, seed=p)
            g.view.view(rpp + 8, K)[:rpp].copy_(X[p * rpp:(p + 1) * rpp])
            srcs.append(g)
        for r in sorted({0, t - 1}):
            for acc in (False, True):
                old = _randn((M, N), seed=r + 5, std=2.0) if acc else None
                og, out = _out(M, N, old if acc else NAN)
                C.gemm_dist(1, [s.view.data_ptr() for s in srcs], [W.data_ptr()], [out.data_ptr()], M, N, K, K,
                            W.stride(0), out.stride(0), b_kmajor, acc, t, r, rpp)
                torch.cuda.synchronize()
                tag = f"mode 1 t{t} r{r} {'nt' if b_kmajor else 'nn'}{' acc' if acc else ''}"
                assert _same(out, _plain(X, W, b_kmajor, old=old)), f"{tag}: differs from the plain GEMM"
                assert _out_intact(og) and all(s.intact() for s in srcs), f"{tag}: wrote outside its views"


@pytest.mark.parametrize("t,rpp", [(1, 64), (2, 192), (4, 64), (4, 256), (8, 192)])
def test_gemm_dist_modes3_and_4_against_fp64(t, rpp):
    """Mode 3: dW[n, H] = dy^T @ concat_p x_p (B gathered along K); mode 4: dW[H, n] = concat_p x_p^T @ dy (A gathered
    along K).  Rank r starts at its own K slice; rank 0's order is the plain GEMM's, so its result is bit-identical."""
    C = _C()
    n, H = 264, 520
    T = t * rpp
    dy = _randn((T, n), t + 3)
    x = _randn((T, H), t + 4)
    xs = [_Guarded(rpp * H, fill=None, seed=p) for p in range(t)]
    for p in range(t):
        xs[p].view.view(rpp, H).copy_(x[p * rpp:(p + 1) * rpp])
    worst = 0.0
    for r in range(t):
        for acc in (False, True):
            for mode in (3, 4):
                M_, N_ = (n, H) if mode == 3 else (H, n)
                old = _randn((M_, N_), seed=r + mode, std=4.0) if acc else None
                og, out = _out(M_, N_, old if acc else NAN)
                if mode == 3:
                    C.gemm_dist(3, [dy.data_ptr()], [s.view.data_ptr() for s in xs], [out.data_ptr()], n, H, T, n, H,
                                out.stride(0), False, acc, t, r, rpp)
                    A, B = dy.t(), x
                else:
                    C.gemm_dist(4, [s.view.data_ptr() for s in xs], [dy.data_ptr()], [out.data_ptr()], H, n, T, H, n,
                                out.stride(0), False, acc, t, r, rpp)
                    A, B = x.t(), dy
                torch.cuda.synchronize()
                tag = f"mode {mode} t{t} rpp{rpp} r{r}{' acc' if acc else ''}"
                assert _out_intact(og) and all(s.intact() for s in xs), f"{tag}: wrote outside its views"
                worst = max(worst, _check_fp64(tag, A, B, out, old))
                if r == 0:
                    want = old.clone() if acc else torch.empty(M_, N_, device="cuda", dtype=BF16)
                    C.gemm(dy if mode == 3 else x, x if mode == 3 else dy, want, True, False, acc, 2)
                    assert _same(out, want), f"{tag}: rank 0 (no K rotation) differs from the plain GEMM"
    print(f"\nmodes 3/4 t{t} rpp{rpp}: element bound c used {worst:.3g} of {ELEM_C}")


def test_k_rotated_bound_rejects_wrong_block_dropped_block_and_two_ulps():
    """The element bound modes 3 and 4 are held to sees a K block of B taken from the wrong place, a K block that
    never arrived (zero) and a 2-ulp error in one element."""
    M, K, N = 520, 1376, 512
    A = _randn((M, K), 1)
    B = _randn((K, N), 2, std=K ** -0.5)
    good = _plain(A, B, False)
    assert _evaluate(A, B, {"k": good})["k"][1] <= ELEM_C
    wrong = B.clone()
    wrong[640:704] = B[704:768]
    dropped = B.clone()
    dropped[640:704] = 0
    for what, Bx in (("wrong block", wrong), ("dropped block", dropped)):
        assert _evaluate(A, B, {"k": _plain(A, Bx, False)})["k"][1] > ELEM_C, f"{what} not rejected"
    i = int(good.float().abs().argmax())
    g2 = good.clone().view(-1)
    g2[i] = (g2[i:i + 1].view(torch.int16) + 2).view(BF16)[0]
    assert _evaluate(A, B, {"k": g2.view(M, N)})["k"][1] > ELEM_C, "2-ulp error not rejected"


# ------------------------------------------------------------------------------------------------------------------
# empty calls
# ------------------------------------------------------------------------------------------------------------------
def test_tp_empty_calls_launch_nothing_and_k0_writes_zeros():
    """gemm_ag, gemm_dist and tp_reduce_parts: M or N = 0 launches nothing; K = 0 writes zeros in overwrite mode and
    leaves C in accumulate mode, as the plain GEMM does."""
    C = _C()
    t, rpp, N = 2, 256, 264
    bufs = [_Guarded(t * rpp * 64, seed=p) for p in range(t)]
    pads = _pads(t)
    pads[0].fill_(3)
    flags = torch.zeros(t * rpp // 256, device="cuda", dtype=torch.int32)
    W = _randn((N, 64), 1)
    torch.cuda.synchronize()
    n0 = _ext.launch_count()
    # gemm_ag: M = 0 (no rows per rank), N = 0
    C.gemm_ag([b.view.data_ptr() for b in bufs], W, torch.empty(0, N, device="cuda", dtype=BF16), True, 0, 0, flags, 1,
              [p.data_ptr() for p in pads], 3, 1)
    C.gemm_ag([b.view.data_ptr() for b in bufs], W[:0], torch.empty(t * rpp, 0, device="cuda", dtype=BF16), True, 0,
              rpp, flags, 1, [p.data_ptr() for p in pads], 3, 1)
    a = _randn((t * rpp, 64), 2)
    for mode in (1, 2, 3, 4):
        C.gemm_dist(mode, [a.data_ptr()] * (t if mode in (1, 4) else 1), [W.data_ptr()] * (t if mode == 3 else 1),
                    [a.data_ptr()] * (t if mode == 2 else 1), 0 if mode < 3 else 64, 0 if mode >= 3 else N,
                    64 if mode < 3 else 0, 64, 64, N, True, False, t, 0, 0)
    C.tp_reduce_parts(torch.empty(t, 0, device="cuda", dtype=BF16), None, torch.empty(0, device="cuda", dtype=BF16))
    torch.cuda.synchronize()
    assert _ext.launch_count() == n0, "an empty call launched a kernel"
    assert bool((pads[1] == 0).all()) and bool((flags == 0).all())
    # K = 0: gemm_ag overwrites with zeros
    og, out = _out(t * rpp, N)
    C.gemm_ag([b.view.data_ptr() for b in bufs], W[:, :0], out, True, 0, rpp, flags, 1, [p.data_ptr() for p in pads],
              3, 1)
    torch.cuda.synchronize()
    assert bool((out == 0).all()) and _out_intact(og)
    # K = 0, mode 2: zeros over every owner's slot; modes 1, 3, 4: zeros, or C unchanged in accumulate mode
    stage = [_Guarded(t * rpp * N, seed=p + 5) for p in range(t)]
    C.gemm_dist(2, [a.data_ptr()], [W.data_ptr()], [s.view.data_ptr() + rpp * N * 2 for s in stage], t * rpp, N, 0, 64,
                64, N, True, False, t, 1, rpp)
    torch.cuda.synchronize()
    for s in stage:
        v = s.view.view(t, rpp, N)
        assert bool((v[1] == 0).all()) and bool(torch.isnan(v[0].float()).all()) and s.intact()
    for mode in (1, 3, 4):
        for acc in (False, True):
            old = _randn((t * rpp, N), 9)
            og, out = _out(t * rpp, N, old)
            rpp_k = rpp if mode == 1 else 0
            C.gemm_dist(mode, [a.data_ptr()] * (t if mode in (1, 4) else 1), [W.data_ptr()] * (t if mode == 3 else 1),
                        [out.data_ptr()], t * rpp, N, 0, 64, 64, out.stride(0), True, acc, t, 0, rpp_k)
            torch.cuda.synchronize()
            want = old if acc else torch.zeros_like(old)
            assert _same(out, want) and _out_intact(og), (mode, acc)


# ------------------------------------------------------------------------------------------------------------------
# refusals: each raises before any launch.  Operands a kernel of the parent code would have dereferenced sit inside
# guarded allocations.
# ------------------------------------------------------------------------------------------------------------------
def _ag_args(t=2, rpp=256, K=64, N=264):
    bufs = [_Guarded(t * rpp * K, seed=p) for p in range(t)]
    pads = _pads(t)
    pads[0].fill_(3)
    return dict(a_bufs=[b.view.data_ptr() for b in bufs], b=_randn((N, K), 1), out=_out(t * rpp, N)[1],
                b_kmajor=True, rank=0, rows_per_peer=rpp, flags=torch.zeros(t * rpp // 256, device="cuda",
                                                                            dtype=torch.int32),
                ag_epoch=1, pads=[p.data_ptr() for p in pads], bar_epoch=3, n_comm=1), (bufs, pads)


def test_gemm_ag_refusals():
    C = _C()
    args, keep = _ag_args()

    def call(**kw):
        return lambda: C.gemm_ag(**{**args, **kw})
    cpu = torch.device("cpu")
    pairs = torch.cuda.get_device_properties(0).multi_processor_count // 2
    _refused(call(a_bufs=args["a_bufs"] * 5), "1..8 ranks")                 # 10 entries: past a host stack array
    _refused(call(pads=args["pads"][:1]), "pads must have 2 entries")      # read past the end of pads
    _refused(call(rank=2), "rank 2 outside")
    _refused(call(rank=-1), "rank -1 outside")
    _refused(call(n_comm=0), "n_comm")
    _refused(call(n_comm=pairs), "n_comm")                                  # no CTA pair left to multiply
    _refused(call(n_comm=pairs + 3), "n_comm")
    _refused(call(ag_epoch=0), "nonzero")
    _refused(call(ag_epoch=1 << 32), "nonzero")
    _refused(call(bar_epoch=0), "nonzero")
    _refused(call(flags=args["flags"].to(cpu)), "flags must be on")
    _refused(call(flags=torch.zeros(4, device="cuda", dtype=torch.int32)[::2]), "flags must be contiguous")
    _refused(call(flags=args["flags"].long()), "flags must be Int")
    _refused(call(flags=torch.zeros(1, device="cuda", dtype=torch.int32)), "flags must hold")
    _refused(call(b=args["b"].to(cpu)), "b must be on")
    _refused(call(b=args["b"].t().contiguous().t()), "b must be 2-D with a contiguous last")
    _refused(call(b=args["b"].float()), "b must be BFloat16")
    _refused(call(out=args["out"].reshape(-1)), "out must be 2-D")
    _refused(call(a_bufs=[args["a_bufs"][0], args["a_bufs"][1] + 2]), "16-byte aligned")
    _refused(call(pads=[args["pads"][0], 0]), "16-byte aligned")


def test_gemm_dist_refusals():
    C = _C()
    t, rpp, K, N = 2, 256, 64, 264
    a = _Guarded(t * rpp * K, fill=0.0)
    w = _Guarded(N * K, fill=0.0)
    st = [_Guarded(t * rpp * N) for _ in range(t)]
    ap, wp = a.view.data_ptr(), w.view.data_ptr()
    cp = [s.view.data_ptr() for s in st]

    def call(mode=2, a_ptrs=(ap,), b_ptrs=(wp,), c_ptrs=tuple(cp), M=t * rpp, nranks=t, rank=0, acc=False, rpp_=rpp):
        return lambda: C.gemm_dist(mode, list(a_ptrs), list(b_ptrs), list(c_ptrs), M, N, K, K, K, N, True, acc,
                                   nranks, rank, rpp_)
    _refused(call(c_ptrs=cp[:1]), "c_ptrs must have 2 entries")            # the epilogue stored through nullptr
    _refused(call(rank=2), "rank 2 outside")                                # m_tile_shift past the tiles
    _refused(call(rank=-1), "rank -1 outside")
    _refused(call(nranks=9, c_ptrs=cp * 4 + cp[:1], M=9 * rpp), "1..8 ranks")
    _refused(call(c_ptrs=cp * 5, nranks=2), "c_ptrs must have 2 entries")   # silently truncated before
    _refused(call(a_ptrs=(ap + 2,)), "a_ptrs must be a 16-byte aligned")
    _refused(call(b_ptrs=(wp + 8,)), "b_ptrs must be a 16-byte aligned")
    _refused(call(c_ptrs=(cp[0], cp[1] + 2)), "c_ptrs must be a 16-byte aligned")
    _refused(call(c_ptrs=(cp[0], 0)), "c_ptrs must be a 16-byte aligned")
    _refused(call(acc=True), "mode 2 overwrites")                           # accumulate was silently ignored
    _refused(call(mode=5), "mode must be 1..4")
    _refused(call(mode=1, a_ptrs=(ap,), c_ptrs=(cp[0],)), "a_ptrs must have 2 entries")
    _refused(call(mode=3, a_ptrs=(ap,), b_ptrs=(wp,), c_ptrs=(cp[0],)), "b_ptrs must have 2 entries")
    _refused(call(mode=4, a_ptrs=(ap, ap, ap), c_ptrs=(cp[0],)), "a_ptrs must have 2 entries")
    _refused(call(mode=1, a_ptrs=(ap, ap), c_ptrs=(cp[0],), M=-256), "negative")


def test_reduce_parts_refusals():
    C = _C()
    t, R, H = 2, 64, 256
    parts = _Guarded(t * R * H + 8, fill=1.0)
    res = _Guarded(2 * R * H + 8, fill=1.0)              # a shorter residual view still reads inside this allocation
    yg = _Guarded(R * H + 8)
    p = parts.view[:t * R * H].view(t, R, H)
    y = yg.view[:R * H].view(R, H)
    cpu = torch.device("cpu")
    _refused(lambda: C.tp_reduce_parts(p, res.view[:(R - 1) * H].view(R - 1, H), y), "residual must have out's shape")
    _refused(lambda: C.tp_reduce_parts(p, res.view[:R * H].view(R, H).float(), y), "residual must be BFloat16")
    _refused(lambda: C.tp_reduce_parts(p, res.view[:R * H].view(R, H).to(cpu), y), "residual must be on")
    _refused(lambda: C.tp_reduce_parts(p, res.view[:2 * R * H].view(R, 2 * H)[:, ::2], y), "residual must be contig")
    _refused(lambda: C.tp_reduce_parts(p, res.view[1:1 + R * H].view(R, H), y), "residual must start")
    _refused(lambda: C.tp_reduce_parts(p, None, torch.empty(R, H, device="cuda")), "out must be BFloat16")
    _refused(lambda: C.tp_reduce_parts(p, None, yg.view[1:1 + R * H].view(R, H)), "out must start")
    _refused(lambda: C.tp_reduce_parts(parts.view[1:1 + t * R * H].view(t, R, H), None, y), "parts must start")
    _refused(lambda: C.tp_reduce_parts(p.to(cpu), None, y), "parts must be on")
    _refused(lambda: C.tp_reduce_parts(p.reshape(t, R * H), None, y), "parts must be")
    _refused(lambda: C.tp_reduce_parts(p[:, :R // 2], None, y), "parts must be")
    assert yg.intact() and res.intact() and parts.intact()
