"""The mixture-of-experts kernels and the grouped GEMM against fp64 on one GPU, at OLMoE's shapes and edges.

Bounds and contracts, none with an outlier budget:

- Grouped GEMM (``gemm_grouped``, modes 0 forward, 1 dgrad, 2 wgrad).  Each expert's block over its padded rows
  ``[seg[e], seg[e+1])`` is bit-identical to the plain GEMM (``gemm(..., variant=1)``, the same single-CTA template,
  K order and epilogue) on the same rows: forward ``trans_b`` against ``W[e]``, dgrad against ``Wt[e]``, wgrad
  ``trans_a`` over the expert's rows, overwrite and accumulate.  Every element also satisfies the bf16 GEMM's bound
  ``|got - exact| <= 2^-8 |exact| + ELEM_C K 2^-24 (|A| @ |B|)`` with K the reduction length (the expert's padded row
  count in wgrad).  Operands sit inside NaN padding and rows of A (and in wgrad of B) at or past ``seg[E]`` are NaN;
  the output is a view inside a buffer of random bits, and nothing outside the expert blocks changes: rows at or past
  ``seg[E]`` keep their bits in forward / dgrad, an empty expert gets exact +0 in overwrite mode and keeps its bits in
  accumulate mode.  The shapes include OLMoE-1B-7B at T 4096 in all six training GEMMs and shapes whose tile order
  takes the grouped L2 rasterisation with a partial last group.
- Routing (``moe_route``).  ``idx`` is the stable top-k of the kernel's own fp32 ``p`` (ties, underflowed zeros
  included, to the lower expert); it agrees with the fp64 order wherever two fp64 probabilities differ by more than
  twice the ``p`` bound; ``w`` is ``p`` at ``idx`` bit for bit; ``|p - p64| <= (24 + E/2 + |l - max l|) 2^-24 p64 +
  2^-126``; and every routing table is exactly the stable counting sort of ``idx``.
- Permute copies rows bit for bit; padding rows are zero.  Combine is within ``2^-8 |y| + k 2^-24 sum |w yp|``; its
  backward's ``dyp`` is ``bf16(w * dy)`` bit for bit and ``dw`` within ``(8 ceil(H / 2048) + 16) 2^-24 sum |dy yp|``.
  The router backward is within ``2^-8 |ref| + 2 (E/32 + 8) 2^-24 p (|dp| + sum p |dp|)`` of fp64
  ``p (dp - sum p dp)``; ``moe_prob_sums`` within ``(T/8 + 8) 2^-24 sum |p|`` of the fp64 column sums.
- ``ops.moe`` end to end with the routing held at the kernel's own choice: y, psum and every gradient against an fp64
  autograd graph, element by element, within a running-error bound (``_path_bound``); a self-test shows the bound
  rejects four wiring mistakes.
- A table entry outside what it indexes is never followed (``moe.cu``): such rows and tokens come out NaN, and every
  byte around the operands keeps its value.

The measured use of each bound is printed (``-s``).
"""
import contextlib
import math
import os
import types

import pytest
import torch
import torch.nn.functional as F

from distributed_training_guide_b200 import _ext
from test_gpu_moe_kernels import _check_layout

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16
U = 2.0 ** -8                 # bf16 unit roundoff
ELEM_C = 1e-2                 # as in test_gpu_gemm_reference.py
PAD = 64                      # elements of NaN / sentinel before and after every operand (keeps 16-byte alignment)
# the end-to-end bound is first order in U; this covers the second-order terms, the fp32 accumulation of every GEMM
# (at most ELEM_C K 2^-24 of a magnitude the bound already counts once, under 2^-10 of it) and the fp32 probabilities
# (2^-16 relative)
PATH_SLACK = 1.05


def _C():
    return _ext.load(required=True)


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _bits(t):
    return t.view(torch.int16) if t.dtype == BF16 else t.view(torch.int32)


# ------------------------------------------------------------------------------------------------------------------
# memory: operands inside NaN padding, outputs inside sentinel buffers
# ------------------------------------------------------------------------------------------------------------------
def _padded(t, fill=float("nan")):
    """A contiguous copy of ``t`` inside a flat buffer with PAD elements of ``fill`` before and after."""
    buf = torch.full((t.numel() + 2 * PAD,), fill, device="cuda", dtype=t.dtype)
    view = buf[PAD:PAD + t.numel()].view(t.shape)
    view.copy_(t)
    return buf, view


def _sentinel(shape, seed=777):
    """A contiguous bf16 view of ``shape`` inside a flat buffer of random bits, PAD elements of them before and
    after."""
    n = math.prod(shape)
    buf = torch.randint(-2 ** 15, 2 ** 15, (n + 2 * PAD,), device="cuda", generator=_gen(seed), dtype=torch.int16)
    return buf.view(BF16), buf.view(BF16)[PAD:PAD + n].view(shape)


def _same_bits(a, b):
    return torch.equal(_bits(a), _bits(b))


# ------------------------------------------------------------------------------------------------------------------
# routings, all through moe_route on constructed logits
# ------------------------------------------------------------------------------------------------------------------
def _route(lg, k):
    p, idx, w, pos, seg, tiles, row_tok, counts = _C().moe_route(lg, k)
    torch.cuda.synchronize()
    return types.SimpleNamespace(lg=lg, k=k, E=lg.shape[1], T=lg.shape[0], p=p, idx=idx, w=w, pos=pos, seg=seg,
                                 tiles=tiles, row_tok=row_tok, counts=counts, segs=seg.tolist(), R=row_tok.numel())


ROUTINGS = ["random", "first-empty", "last-empty", "one-expert", "no-padding", "T1"]


def _routing_logits(kind, T, E, k, seed=0):
    """Logits [T, E] (bf16) and k for a routing kind: random; expert 0 or E-1 never chosen; every token on one
    expert (k 1, so every other expert is empty and one segment spans many tiles); every count a multiple of 128
    (T k = 128 E, no padding row); one token."""
    if kind == "T1":
        T = 1
    lg = torch.randn(T, E, device="cuda", generator=_gen(seed))
    if kind == "first-empty":
        lg[:, 0] = -30.0
    elif kind == "last-empty":
        lg[:, E - 1] = -30.0
    elif kind == "one-expert":
        k = 1
        lg[:, E // 2] = 30.0
    elif kind == "no-padding":
        assert T * k == 128 * E and E % k == 0
        t = torch.arange(T, device="cuda")
        grp = t % (E // k)                                         # token t takes experts k grp .. k grp + k - 1
        lg = 0.1 * lg
        for s in range(k):
            lg[t, k * grp + s] = 5.0 - s
    return lg.to(BF16), k


# ------------------------------------------------------------------------------------------------------------------
# grouped GEMM
# ------------------------------------------------------------------------------------------------------------------
def _group_m(num_m_tiles, K):
    """The launcher's grouped-rasterisation rule (gemm_wgmma.cu, launch_gemm): row tiles per L2 group, 0 = none."""
    budget = int(os.environ.get("DTG_GEMM_L2_BUDGET_MB", "16")) << 20
    gm = max(budget // (128 * K * 2), 8)
    return 0 if gm >= num_m_tiles else gm


def _elem_c(got, exact, mag, K):
    """The least c with |got - exact| <= 2^-8 |exact| + c K 2^-24 mag over the block (inf for a NaN)."""
    bound = (mag.double() * (K * 2.0 ** -24)).clamp_min_(1e-300)
    r = ((got.double() - exact).abs_() - exact.abs() * U) / bound
    r = torch.where(torch.isnan(r), torch.full_like(r, float("inf")), r)
    return r.max().item()


def _abs_product(a, b):
    """|a| @ |b| for bf16 a, b: a bf16 product with fp32 accumulation, rounded once to bf16, so the accumulation term
    of the bound is within 2^-8 of its exact value."""
    prev = torch.backends.cuda.matmul.allow_bf16_reduced_precision_reduction
    torch.backends.cuda.matmul.allow_bf16_reduced_precision_reduction = False
    try:
        return torch.matmul(a.abs(), b.abs()).float()
    finally:
        torch.backends.cuda.matmul.allow_bf16_reduced_precision_reduction = prev


def _fwd_dgrad_case(tag, mode, r, N, K, seed):
    """gemm_grouped mode 0 (b = W [E, N, K]) or 1 (b = Wt [E, K, N]) over the routing r; returns the largest c."""
    C = _C()
    E, R, segs = r.E, r.R, r.segs
    used = segs[-1]
    g = _gen(seed)
    a = torch.randn(R, K, device="cuda", generator=g).to(BF16)
    a[used:] = float("nan")                                        # rows past the last segment: never read into C
    b = (torch.randn((E, N, K) if mode == 0 else (E, K, N), device="cuda", generator=g) / math.sqrt(K)).to(BF16)
    _, A = _padded(a)
    _, B = _padded(b)
    buf, out = _sentinel((R, N))
    out[:used] = float("nan")
    before = buf.clone()
    C.gemm_grouped(mode, A, B, out, r.seg, r.tiles)
    mask = torch.ones_like(buf, dtype=torch.bool)
    mask[PAD:PAD + used * N] = False
    assert torch.equal(_bits(buf)[mask], _bits(before)[mask]), f"{tag}: wrote outside rows [0, seg[E])"
    worst = 0.0
    for e in range(E):
        s0, s1 = segs[e], segs[e + 1]
        if s1 == s0:
            continue
        plain = torch.empty(s1 - s0, N, device="cuda", dtype=BF16)
        C.gemm(A[s0:s1], B[e], plain, False, mode == 0, False, 1)
        assert _same_bits(out[s0:s1], plain), f"{tag}: expert {e} differs from the plain GEMM"
        Bl = B[e].t() if mode == 0 else B[e]                       # [K, N]
        exact = A[s0:s1].double() @ Bl.double()
        worst = max(worst, _elem_c(out[s0:s1], exact, _abs_product(A[s0:s1], Bl), K))
        del exact
    again_buf, again = _sentinel((R, N), seed=778)
    C.gemm_grouped(mode, A, B, again, r.seg, r.tiles)
    assert _same_bits(again[:used], out[:used]), f"{tag}: not bit-identical on a repeat"
    assert worst <= ELEM_C, f"{tag}: an element needs c = {worst:.3g} > {ELEM_C}"
    return worst


def _wgrad_case(tag, r, M, N, seed):
    """gemm_grouped mode 2: dW_e [M, N] (+)= a[seg_e]^T b[seg_e], overwrite then accumulate; returns the largest c."""
    C = _C()
    E, R, segs = r.E, r.R, r.segs
    used = segs[-1]
    g = _gen(seed)
    a = torch.randn(R, M, device="cuda", generator=g).to(BF16)
    b = torch.randn(R, N, device="cuda", generator=g).to(BF16)
    a[used:] = float("nan")                                        # any read past seg[E] would poison dW
    b[used:] = float("nan")
    _, A = _padded(a)
    _, B = _padded(b)
    worst = 0.0
    for acc in (False, True):
        buf, out = _sentinel((E, M, N), seed=900 + acc)
        if acc:
            out.copy_((torch.randn(E, M, N, device="cuda", generator=g) * 8).to(BF16))
            for e in range(E):
                if segs[e + 1] == segs[e]:
                    out[e] = float("nan")                          # an empty expert keeps even NaN and -0
                    out[e, 0, 0] = -0.0
        else:
            out.fill_(float("nan"))
        old = out.clone()
        before = buf.clone()
        C.gemm_grouped(2, A, B, out, r.seg, None, acc)
        mask = torch.ones_like(buf, dtype=torch.bool)
        mask[PAD:PAD + E * M * N] = False
        assert torch.equal(_bits(buf)[mask], _bits(before)[mask]), f"{tag}: wrote outside dW"
        for e in range(E):
            s0, s1 = segs[e], segs[e + 1]
            if s1 == s0:
                if acc:
                    assert _same_bits(out[e], old[e]), f"{tag}: empty expert {e} changed in accumulate mode"
                else:
                    assert bool((_bits(out[e]) == 0).all()), f"{tag}: empty expert {e} is not +0"
                continue
            plain = old[e].clone()
            C.gemm(A[s0:s1], B[s0:s1], plain, True, False, acc, 1)
            assert _same_bits(out[e], plain), f"{tag} acc={acc}: expert {e} differs from the plain GEMM"
            exact = A[s0:s1].double().t() @ B[s0:s1].double()
            mag = _abs_product(A[s0:s1].t(), B[s0:s1])
            if acc:
                exact += old[e].double()
                mag += old[e].float().abs()
            worst = max(worst, _elem_c(out[e], exact, mag, s1 - s0))
            del exact, mag
    assert worst <= ELEM_C, f"{tag}: an element needs c = {worst:.3g} > {ELEM_C}"
    return worst


DEBUG = dict(E=8, k=2, H=256, I=128, T=512)
OLMOE = dict(E=64, k=8, H=2048, I=1024, T=4096)


def _training_gemms(H, I):
    """The six grouped GEMMs of one MoE layer's step: (name, mode, N or M, K or N)."""
    return [("fwd-gate_up", 0, 2 * I, H), ("fwd-down", 0, H, I), ("dgrad-down", 1, I, H),
            ("dgrad-gate_up", 1, H, 2 * I), ("wgrad-down", 2, H, I), ("wgrad-gate_up", 2, 2 * I, H)]


def _run_gemm(tag, mode, r, d0, d1, seed):
    c = _wgrad_case(tag, r, d0, d1, seed) if mode == 2 else _fwd_dgrad_case(tag, mode, r, d0, d1, seed)
    print(f"\n{tag}: bit-identical to the plain GEMM per expert; element c {c:.3g} (bound {ELEM_C})")


@pytest.mark.parametrize("kind", ROUTINGS)
def test_grouped_gemm_debug_olmoe_routings(kind):
    d = DEBUG
    lg, k = _routing_logits(kind, d["T"], d["E"], d["k"], seed=1)
    r = _route(lg, k)
    _check_layout(r.idx, r.E, r.pos, r.seg, r.tiles, r.row_tok, r.counts)
    if kind == "first-empty":
        assert r.segs[1] == 0
    if kind == "last-empty":
        assert r.segs[-1] == r.segs[-2]
    if kind == "one-expert":
        assert r.counts.tolist().count(0) == r.E - 1 and r.segs[-1] >= 4 * 128
    if kind == "no-padding":
        assert r.segs == [128 * e for e in range(r.E + 1)]
    for i, (name, mode, a, b) in enumerate(_training_gemms(d["H"], d["I"])):
        _run_gemm(f"debug {kind} {name}", mode, r, a, b, seed=10 + i)


@pytest.mark.parametrize("name,mode,d0,d1", _training_gemms(OLMOE["H"], OLMOE["I"]))
def test_grouped_gemm_olmoe_1b_7b(name, mode, d0, d1):
    d = OLMOE
    r = _route(torch.randn(d["T"], d["E"], device="cuda", generator=_gen(5)).to(BF16), d["k"])
    R = r.R
    assert R == 40960
    # both tile orders take the grouped L2 rasterisation at this geometry
    assert _group_m(R // 128, d1) > 0 if mode < 2 else _group_m(d0 // 128, R) > 0
    _run_gemm(f"OLMoE-1B-7B {name}", mode, r, d0, d1, seed=20 + mode)
    torch.cuda.empty_cache()


def test_grouped_gemm_partial_l2_groups():
    """T 4000 at E 64, k 8 gives 314 row tiles: forward at K 2048 runs groups of 32 row tiles, the last of 26; wgrad
    at M 1408 (11 row tiles) over those 40192 rows runs groups of 8, the last of 3."""
    r = _route(torch.randn(4000, 64, device="cuda", generator=_gen(6)).to(BF16), 8)
    tiles = r.R // 128
    gm = _group_m(tiles, 2048)
    assert gm > 0 and tiles % gm != 0, (tiles, gm)
    _run_gemm("partial-group fwd K2048 N256", 0, r, 256, 2048, seed=30)
    _run_gemm("partial-group dgrad K2048 N256", 1, r, 256, 2048, seed=31)
    gm2 = _group_m(1408 // 128, r.R)
    assert gm2 > 0 and (1408 // 128) % gm2 != 0, gm2
    _run_gemm("partial-group wgrad M1408 N256", 2, r, 1408, 256, seed=32)


# (mode, N or M, K or N): a forward K tail, N below, off and past the 256-column tile in every mode, wgrad N < 256
EDGES = [(0, 256, 200), (0, 8, 256), (0, 136, 256), (0, 384, 128), (0, 1000, 64), (1, 8, 256), (1, 136, 128),
         (1, 384, 64), (1, 1000, 256), (2, 128, 8), (2, 256, 136), (2, 128, 384), (2, 256, 1000)]


@pytest.mark.parametrize("kind", ["random", "first-empty", "last-empty"])
@pytest.mark.parametrize("mode,d0,d1", EDGES)
def test_grouped_gemm_edges(mode, d0, d1, kind):
    lg, k = _routing_logits(kind, 512, 8, 2, seed=2)
    _run_gemm(f"edge {kind} mode {mode} {d0}x{d1}", mode, _route(lg, k), d0, d1, seed=40 + d0 + d1)


# ------------------------------------------------------------------------------------------------------------------
# routing
# ------------------------------------------------------------------------------------------------------------------
def _p_bound(lg, p64):
    l = lg.double()
    span = l.max(-1, keepdim=True).values - l
    E = lg.shape[1]
    return (24 + E / 2 + span) * 2.0 ** -24 * p64 + 2.0 ** -126


def _check_route_contract(lg, k, tag):
    """Kernel routing against its own p (tie rule), fp64 (order and p bound) and the layout, exactly."""
    r = _route(lg, k)
    T, E = lg.shape
    p, idx = r.p, r.idx.long()
    stable = torch.sort(-p, dim=-1, stable=True).indices[:, :k]
    assert torch.equal(idx, stable), f"{tag}: idx is not the stable top-k of the kernel's p"
    assert _same_bits(r.w, p.gather(1, idx)), f"{tag}: w is not p at idx"
    p64 = torch.softmax(lg.double(), -1)
    pb = _p_bound(lg, p64)
    use = ((p.double() - p64).abs() / pb).max().item()
    assert use <= 1.0, f"{tag}: p needs {use:.3g} of its bound"
    # fp64 order: no expert still available at slot s beats the one picked by more than the two p bounds
    avail = torch.ones(T, E, dtype=torch.bool, device="cuda")
    for s in range(k):
        pick = idx[:, s:s + 1]
        best = torch.where(avail, p64 - pb, torch.full_like(p64, -1.0)).max(-1, keepdim=True).values
        assert bool(((p64 + pb).gather(1, pick) >= best).all()), f"{tag}: slot {s} contradicts the fp64 order"
        avail.scatter_(1, pick, False)
    _check_layout(r.idx, E, r.pos, r.seg, r.tiles, r.row_tok, r.counts)
    print(f"\nroute {tag}: p uses {use:.3g} of its bound")
    return r


# T across the 32-token chunks, and a long serial scan at OLMoE's E and with all 8 lanes of experts filled
@pytest.mark.parametrize("T,E,k", [(T, E, k) for E, k in [(64, 8), (33, 5), (255, 7), (256, 8), (8, 8), (1, 1)]
                                   for T in (31, 32, 33)] + [(131072, 64, 8), (131072, 256, 8)])
def test_route_against_fp64(T, E, k):
    lg = (torch.randn(T, E, device="cuda", generator=_gen(T + E)) * 3).to(BF16)
    _check_route_contract(lg, k, f"T{T} E{E} k{k}")


def test_route_underflow_rows_and_ties():
    """Rows whose logits span more than ~104: every expert but one has an fp32 probability of exactly 0, fp64 ranks
    them by their logits, the kernel by index.  All-equal rows tie everywhere."""
    T, E, k = 96, 64, 8
    lg = torch.randn(T, E, device="cuda", generator=_gen(3))
    lg[0:32] = -120.0 + 0.25 * torch.arange(E, device="cuda")     # fp64 prefers the highest index
    lg[0:32, 17] = 10.0                                            # the one nonzero probability
    lg[32:64] = 0.0                                                # all tied
    lg[48:64, ::2] = 2.0                                           # 32 tied at the top
    r = _check_route_contract(lg.to(BF16), k, "underflow")
    p = r.p[0:32]
    assert bool((p.gt(0).sum(-1) == 1).all())
    assert r.idx[0].tolist() == [17] + list(range(7))
    assert r.idx[32].tolist() == list(range(8)) and r.idx[48].tolist() == list(range(0, 16, 2))


def test_route_strided_logits():
    T, E, k = 1000, 64, 8
    full = torch.randn(T, E + 40, device="cuda", generator=_gen(4)).to(BF16)
    lg = full[:, 3:3 + E]
    assert lg.stride(0) == E + 40 and lg.stride(1) == 1
    a = _check_route_contract(lg, k, "strided")
    b = _route(lg.contiguous(), k)
    for name in ("p", "idx", "w", "pos", "seg", "tiles", "counts"):
        assert torch.equal(getattr(a, name), getattr(b, name)), name


# ------------------------------------------------------------------------------------------------------------------
# permute, combine, their backwards, the router backward and the probability sums
# ------------------------------------------------------------------------------------------------------------------
@contextlib.contextmanager
def _prefilled(nbytes, fill_bits):
    """Inside a fresh memory pool, leave a freed block of ``nbytes`` filled with ``fill_bits``: the first allocation
    the binding makes gets it, so rows its kernel does not write keep these bits.  Yields the block's address."""
    pool = torch.cuda.MemPool()
    with torch.cuda.use_mem_pool(pool):
        t = torch.full((nbytes // 2,), fill_bits, device="cuda", dtype=torch.int16)
        ptr = t.data_ptr()
        del t
        yield ptr


SENT = 0x3F9D   # bf16 1.2265625: a sentinel no kernel writes


@pytest.mark.parametrize("H", [8, 136, 2048])
@pytest.mark.parametrize("kind", ["random", "first-empty", "one-expert", "no-padding"])
def test_permute_bit_exact(kind, H):
    lg, k = _routing_logits(kind, 512, 8, 2, seed=7)
    r = _route(lg, k)
    x = torch.randn(r.T, H, device="cuda", generator=_gen(H)).to(BF16)
    with _prefilled(r.R * H * 2, SENT) as ptr:
        xp = _C().moe_permute(x, r.row_tok, r.seg, k)
    assert xp.data_ptr() == ptr
    used = r.segs[-1]
    rt = r.row_tok[:used].long()
    real = rt >= 0
    assert _same_bits(xp[:used][real], x[rt[real] // k])
    assert bool((_bits(xp[:used][~real]) == 0).all())
    assert bool((_bits(xp[used:]) == SENT).all()), "rows past seg[E] were written"


@pytest.mark.parametrize("k", [1, 2, 8])
@pytest.mark.parametrize("H", [8, 136, 2048])
def test_combine_against_fp64(k, H):
    C = _C()
    r = _route(torch.randn(300, 16, device="cuda", generator=_gen(k)).to(BF16), k)
    yp = torch.randn(r.R, H, device="cuda", generator=_gen(H)).to(BF16)
    pos = r.pos.long()
    worst = 0.0
    for w in (r.w, None):
        y = C.moe_combine(yp, r.pos, w)
        wd = w.double() if w is not None else torch.ones(r.T, k, device="cuda", dtype=torch.float64)
        terms = wd[:, :, None] * yp.double()[pos]
        ref = terms.sum(1)
        bound = U * ref.abs() + k * 2.0 ** -24 * terms.abs().sum(1)
        use = ((y.double() - ref).abs() / bound.clamp_min(1e-300)).max().item()
        assert use <= 1.0, (w is None, use)
        worst = max(worst, use)
    # a NaN weight reaches exactly its token's row
    wn = r.w.clone()
    wn[17, k - 1] = float("nan")
    y0, y1 = C.moe_combine(yp, r.pos, r.w), C.moe_combine(yp, r.pos, wn)
    assert bool(torch.isnan(y1[17]).all())
    others = torch.arange(r.T, device="cuda") != 17
    assert _same_bits(y1[others], y0[others])
    print(f"\ncombine k{k} H{H}: {worst:.3g} of the bound")


@pytest.mark.parametrize("H", [8, 136, 2048])
def test_combine_backward_against_fp64(H):
    C = _C()
    k = 8
    r = _route(torch.randn(333, 64, device="cuda", generator=_gen(H)).to(BF16), k)
    yp = torch.randn(r.R, H, device="cuda", generator=_gen(1)).to(BF16)
    dy = torch.randn(r.T, H, device="cuda", generator=_gen(2)).to(BF16)
    with _prefilled(r.R * H * 2, SENT) as ptr:
        dyp, dw = C.moe_combine_bwd(dy, yp, r.row_tok, r.seg, r.w)
    assert dyp.data_ptr() == ptr
    used = r.segs[-1]
    rt = r.row_tok[:used].long()
    real = rt >= 0
    want = (r.w.reshape(-1)[rt[real], None] * dy[rt[real] // k].float()).to(BF16)
    assert _same_bits(dyp[:used][real], want)
    assert bool((_bits(dyp[:used][~real]) == 0).all())
    assert bool((_bits(dyp[used:]) == SENT).all())
    prod = dy.double()[:, None, :] * yp.double()[r.pos.long()]
    ref, mag = prod.sum(-1), prod.abs().sum(-1)
    bound = (8 * math.ceil(H / 2048) + 16) * 2.0 ** -24 * mag
    use = ((dw.double() - ref).abs() / bound.clamp_min(1e-300)).max().item()
    assert use <= 1.0, use
    print(f"\ncombine backward H{H}: dyp bit-identical, dw {use:.3g} of the bound")


@pytest.mark.parametrize("E,k", [(8, 2), (64, 8), (256, 8)])
@pytest.mark.parametrize("with_dpsum", [False, True])
def test_router_backward_against_fp64(E, k, with_dpsum):
    C = _C()
    T = 500
    r = _route(torch.randn(T, E, device="cuda", generator=_gen(E)).to(BF16), k)
    dw = torch.randn(T, k, device="cuda", generator=_gen(1)) * 10
    dpsum = torch.randn(E, device="cuda", generator=_gen(2)) * 10 if with_dpsum else None
    dl = C.moe_router_bwd(r.p, r.idx, dw, dpsum)
    p = r.p.double()
    dp = torch.zeros(T, E, device="cuda", dtype=torch.float64) if dpsum is None else dpsum.double()[None].repeat(T, 1)
    dp.scatter_add_(1, r.idx.long(), dw.double())
    ref = p * (dp - (p * dp).sum(-1, keepdim=True))
    bound = U * ref.abs() + 2 * (E / 32 + 8) * 2.0 ** -24 * p * (dp.abs() + (p * dp.abs()).sum(-1, keepdim=True))
    use = ((dl.double() - ref).abs() / bound.clamp_min(1e-300)).max().item()
    assert use <= 1.0, use
    if with_dpsum:   # the dpsum term is large enough that ignoring it breaks the bound
        no = p * (dp - dpsum.double() - (p * (dp - dpsum.double())).sum(-1, keepdim=True))
        assert ((no - ref).abs() > bound).any()
    print(f"\nrouter backward E{E} dpsum={with_dpsum}: {use:.3g} of the bound")


@pytest.mark.parametrize("T,E", [(1, 8), (333, 64), (4096, 64), (70000, 256)])
def test_prob_sums_against_fp64(T, E):
    p = torch.softmax(torch.randn(T, E, device="cuda", generator=_gen(T)) * 2, -1)
    got = _C().moe_prob_sums(p)
    ref = p.double().sum(0)
    bound = (T / 8 + 8) * 2.0 ** -24 * p.double().abs().sum(0)
    use = ((got.double() - ref).abs() / bound).max().item()
    assert use <= 1.0, use
    print(f"\nprob sums T{T} E{E}: {use:.3g} of the bound")


# ------------------------------------------------------------------------------------------------------------------
# ops.moe end to end with the routing held fixed
# ------------------------------------------------------------------------------------------------------------------
MUTATIONS = ("swap-gate-up", "drop-slot", "no-dpsum", "no-router-dx")


def moe_fixed_ref(x, gate_w, gate_up, down, idx, logits=None, mutate=None):
    """ops.moe as an autograd graph in the inputs' dtype with the experts ``idx`` [T, k] held fixed:
    ``y = sum_slot p[t, idx] expert_idx(x_t)`` with ``p = softmax(logits)``.  With ``logits`` (the kernel's bf16
    router logits) the graph's logits are ``x gate_w^T + (logits - x gate_w^T).detach()``: the kernel's values with the
    exact gradient.  ``mutate`` names a wiring mistake the bound must reject (the self-test).  Returns (y, psum)."""
    lin = (x.detach() if mutate == "no-router-dx" else x) @ gate_w.t()
    lg = lin if logits is None else lin + (logits.to(lin.dtype) - lin).detach()
    p = torch.softmax(lg, -1)
    T, k = idx.shape
    y = torch.zeros_like(x)
    for e in range(gate_w.shape[0]):
        tok, slot = (idx == e).nonzero(as_tuple=True)
        if mutate == "drop-slot":
            tok = tok[slot != k - 1]
        if tok.numel() == 0:
            continue
        g, u = (x[tok] @ gate_up[e].t()).chunk(2, dim=-1)
        if mutate == "swap-gate-up":
            g, u = u, g
        ye = (F.silu(g) * u) @ down[e].t()
        y = y.index_add(0, tok, ye * p[tok, e, None])
    return y, p.sum(0)


def moe_fixed_grads(x, gate_w, gate_up, down, idx, dy, dpsum, logits=None, mutate=None, dtype=torch.float64):
    """y, psum and the gradients (dx, d_gate, d_gate_up, d_down) of ``moe_fixed_ref`` in ``dtype`` for the upstream
    gradients dy [T, H] and dpsum [E]."""
    leaves = [t.detach().to(dtype).requires_grad_() for t in (x, gate_w, gate_up, down)]
    y, psum = moe_fixed_ref(*leaves, idx, logits=logits, mutate=mutate)
    dps = torch.zeros_like(psum) if mutate == "no-dpsum" else dpsum.to(dtype)
    grads = torch.autograd.grad((y, psum), leaves, (dy.to(dtype), dps))
    return (y.detach(), psum.detach()) + tuple(grads)


def _path_bound(x, gate_w, gate_up, down, idx, p, dy, dpsum, dtype):
    """Values and first-order error bounds, in units of U, of the kernel path's outputs (y, dx, d_gate, d_gate_up,
    d_down).  Every bf16 rounding the path makes (gu, h, yp, y, dyp, dh, dgu, dxp, the combined dx, dlogits, dx, and
    every weight gradient) adds U times the magnitude of the rounded value, and the error reaching a value from its
    inputs is propagated with the absolute value of each operation (|A| @ M for a product, |silu'| and |silu''| for
    the SwiGLU and its backward).  The router logits are taken as the kernel rounded them, so they carry no error.
    Computed per expert like the kernels, in ``dtype`` (fp32 is ample for a bound; fp64 lets a test compare the
    values with autograd).  Returns {name: (value, bound)}."""
    T, H = x.shape
    E, k = gate_w.shape[0], idx.shape[1]
    X = x.to(dtype)
    P = p.to(dtype)
    DY = dy.to(dtype)
    z = lambda *s: torch.zeros(*s, device=x.device, dtype=dtype)
    Y, MY, dX1, MdX1 = z(T, H), z(T, H), z(T, H), z(T, H)
    dW, MdW = z(T, k), z(T, k)
    dGU, MdGU = z(*gate_up.shape), z(*gate_up.shape)
    dDN, MdDN = z(*down.shape), z(*down.shape)
    for e in range(E):
        tok, slot = (idx == e).nonzero(as_tuple=True)
        if tok.numel() == 0:
            continue
        Gw, Dw = gate_up[e].to(dtype), down[e].to(dtype)
        xe = X[tok]
        gu = xe @ Gw.t()
        g, u = gu.chunk(2, -1)
        Mg, Mu = g.abs(), u.abs()
        sg = torch.sigmoid(g)
        s0 = g * sg
        s1 = sg * (1 + g * (1 - sg))
        s2 = sg * (1 - sg) * (2 + g * (1 - 2 * sg))
        h = s0 * u
        Mh = h.abs() + (s1 * u).abs() * Mg + s0.abs() * Mu
        yp = h @ Dw.t()
        Myp = yp.abs() + Mh @ Dw.abs().t()
        we = P[tok, e][:, None]
        Y.index_add_(0, tok, we * yp)
        MY.index_add_(0, tok, we * Myp)
        dye = DY[tok]
        dyp = we * dye
        Mdyp = dyp.abs()
        dW[tok, slot] = (dye * yp).sum(-1)
        MdW[tok, slot] = (dye.abs() * Myp).sum(-1)
        dh = dyp @ Dw
        Mdh = dh.abs() + Mdyp @ Dw.abs()
        dg, du = dh * u * s1, dh * s0
        Mdg = dg.abs() + (u * s1).abs() * Mdh + dh.abs() * (s1.abs() * Mu + (u * s2).abs() * Mg)
        Mdu = du.abs() + s0.abs() * Mdh + dh.abs() * s1.abs() * Mg
        dgu, Mdgu = torch.cat([dg, du], -1), torch.cat([Mdg, Mdu], -1)
        dxp = dgu @ Gw
        dX1.index_add_(0, tok, dxp)
        MdX1.index_add_(0, tok, dxp.abs() + Mdgu @ Gw.abs())
        dDN[e] = dyp.t() @ h
        MdDN[e] = dDN[e].abs() + Mdyp.t() @ h.abs() + dyp.abs().t() @ Mh
        dGU[e] = dgu.t() @ xe
        MdGU[e] = dGU[e].abs() + Mdgu.t() @ xe.abs()
    MY += Y.abs()
    MdX1 += dX1.abs()
    dp = dpsum.to(dtype)[None].repeat(T, 1).scatter_add_(1, idx.long(), dW)
    Mdp = z(T, E).scatter_add_(1, idx.long(), MdW)
    dl = P * (dp - (P * dp).sum(-1, keepdim=True))
    Mdl = dl.abs() + P * (Mdp + (P * Mdp).sum(-1, keepdim=True))
    GW = gate_w.to(dtype)
    dX = dX1 + dl @ GW
    MdX = dX.abs() + MdX1 + Mdl @ GW.abs()
    dG = dl.t() @ X
    MdG = dG.abs() + Mdl.t() @ X.abs()
    return {"y": (Y, MY), "dx": (dX, MdX), "d_gate": (dG, MdG), "d_gate_up": (dGU, MdGU), "d_down": (dDN, MdDN)}


def _moe_inputs(E, k, H, I, T, seed):
    g = _gen(seed)
    x = torch.randn(T, H, device="cuda", generator=g).to(BF16)
    gate_w = (torch.randn(E, H, device="cuda", generator=g) / math.sqrt(H)).to(BF16)
    gate_up = (torch.randn(E, 2 * I, H, device="cuda", generator=g) / math.sqrt(H)).to(BF16)
    down = (torch.randn(E, H, I, device="cuda", generator=g) / math.sqrt(I)).to(BF16)
    dy = torch.randn(T, H, device="cuda", generator=g).to(BF16)
    dpsum = torch.randn(E, device="cuda", generator=g) * math.sqrt(H)   # an aux term c sum_e psum_e r_e, c = sqrt(H)
    return x, gate_w, gate_up, down, dy, dpsum


def _kernel_moe(x, gate_w, gate_up, down, k, dy, dpsum):
    from distributed_training_guide_b200 import ops

    leaves = [t.clone().requires_grad_() for t in (x, gate_w, gate_up, down)]
    n0 = _ext.launch_count()
    y, psum, counts = ops.moe(*leaves, k)
    grads = torch.autograd.grad((y, psum), leaves, (dy, dpsum))
    assert _ext.launch_count() > n0, "ops.moe did not run the sm_90a kernels"
    return (y.detach(), psum.detach()) + tuple(grads)


NAMES = ("y", "psum", "dx", "d_gate", "d_gate_up", "d_down")


@pytest.mark.parametrize("geometry", ["debug-olmoe", "OLMoE-1B-7B"])
def test_ops_moe_fixed_routing_against_fp64(geometry):
    from distributed_training_guide_b200 import ops

    d = DEBUG if geometry == "debug-olmoe" else OLMOE
    E, k, H, I, T = d["E"], d["k"], d["H"], d["I"], d["T"]
    x, gate_w, gate_up, down, dy, dpsum = _moe_inputs(E, k, H, I, T, seed=11)
    logits = ops.gemm(x, gate_w, trans_b=True)                     # what _MoE computes, bit for bit
    r = _route(logits, k)
    got = dict(zip(NAMES, _kernel_moe(x, gate_w, gate_up, down, k, dy, dpsum)))
    ref = dict(zip(NAMES, moe_fixed_grads(x, gate_w, gate_up, down, r.idx, dy, dpsum, logits=logits)))
    bounds = _path_bound(x, gate_w, gate_up, down, r.idx, r.p, dy, dpsum, torch.float32)
    report = []
    for name in ("y", "dx", "d_gate", "d_gate_up", "d_down"):
        b = bounds[name][1].double() * (U * PATH_SLACK)
        err = (got[name].double() - ref[name]).abs()
        use = torch.where(torch.isnan(err), torch.full_like(err, float("inf")), err / b.clamp_min(1e-300)).max().item()
        report.append(f"{name} {use:.3g}")
        assert use <= 1.0, f"{geometry} {name}: an element needs {use:.3g} of the bound"
    p64 = torch.softmax(logits.double(), -1)
    pb = _p_bound(logits, p64).sum(0) + (T / 8 + 8) * 2.0 ** -24 * p64.sum(0)
    use = ((got["psum"].double() - ref["psum"]).abs() / pb).max().item()
    report.append(f"psum {use:.3g}")
    assert use <= 1.0, f"{geometry} psum: {use:.3g} of the bound"
    print(f"\nops.moe {geometry} fixed routing, bound use: " + ", ".join(report))
    if geometry != "debug-olmoe":
        return
    # self-test: the bound rejects each wiring mistake, made in the reference
    for m in MUTATIONS:
        bad = dict(zip(NAMES, moe_fixed_grads(x, gate_w, gate_up, down, r.idx, dy, dpsum, logits=logits, mutate=m)))
        caught = [n for n in ("y", "dx", "d_gate", "d_gate_up", "d_down")
                  if ((got[n].double() - bad[n]).abs() > bounds[n][1].double() * (U * PATH_SLACK)).any()]
        print(f"mutation {m}: rejected by {caught}")
        assert caught, f"the bound does not reject {m}"


def test_ops_moe_is_bit_identical_run_to_run():
    d = DEBUG
    x, gate_w, gate_up, down, dy, dpsum = _moe_inputs(d["E"], d["k"], d["H"], d["I"], d["T"], seed=12)
    a = _kernel_moe(x, gate_w, gate_up, down, d["k"], dy, dpsum)
    b = _kernel_moe(x, gate_w, gate_up, down, d["k"], dy, dpsum)
    for n, u, v in zip(NAMES, a, b):
        assert _same_bits(u, v), n


def test_ops_moe_flat_buffer_micro_batches():
    """Weight gradients through _emit_weight_grad into flat-buffer views: the first micro-batch overwrites, the second
    accumulates, and an expert the second sends no token keeps the first one's gradient bit for bit."""
    from distributed_training_guide_b200 import ops

    d = DEBUG
    E, k, H, I, T = d["E"], d["k"], d["H"], d["I"], d["T"]
    x1, gate_w, gate_up, down, dy1, dpsum1 = _moe_inputs(E, k, H, I, T, seed=13)
    gate_w[0] = 0.5 / math.sqrt(H)                                 # expert 0's logit is 0.5 sqrt(H) mean(x)
    x2, _, _, _, dy2, dpsum2 = _moe_inputs(E, k, H, I, T, seed=14)
    x2 = (x2.float() - 3).to(BF16)                                 # ... -24 in the second micro-batch: never chosen
    assert int(_route(ops.gemm(x1, gate_w, trans_b=True), k).counts[0]) > 0
    assert int(_route(ops.gemm(x2, gate_w, trans_b=True), k).counts[0]) == 0
    plain = [_kernel_moe(x, gate_w, gate_up, down, k, dy, dps)[3:] for x, dy, dps in ((x1, dy1, dpsum1),
                                                                                     (x2, dy2, dpsum2))]
    flat = torch.full((gate_w.numel() + gate_up.numel() + down.numel() + 2 * PAD,), float("nan"), device="cuda",
                      dtype=BF16)
    params = [t.clone().requires_grad_() for t in (gate_w, gate_up, down)]
    off = PAD
    for prm in params:
        prm._dtg_grad = flat[off:off + prm.numel()].view(prm.shape)
        off += prm.numel()
    after = []
    for x, dy, dps in ((x1, dy1, dpsum1), (x2, dy2, dpsum2)):
        xl = x.clone().requires_grad_()
        y, psum, _ = ops.moe(xl, *params, k)
        torch.autograd.backward((y, psum), (dy, dps))
        assert all(prm.grad is None for prm in params)
        after.append([prm._dtg_grad.clone() for prm in params])
    assert all(prm._dtg_writes == 2 for prm in params)
    assert bool(torch.isnan(flat[:PAD]).all()) and bool(torch.isnan(flat[off:]).all())
    for i, name in enumerate(("d_gate", "d_gate_up", "d_down")):
        assert _same_bits(after[0][i], plain[0][i]), f"{name}: the first micro-batch differs from a plain run"
        g1, g2, acc = plain[0][i].double(), plain[1][i].double(), after[1][i].double()
        bound = U * (g1 + g2).abs() + U * g2.abs() + 2.0 ** -24 * (g1.abs() + g2.abs()) * H
        assert bool(((acc - (g1 + g2)).abs() <= bound * 1.01).all()), f"{name}: accumulate"
    for i in (1, 2):                                               # expert 0 got no token in the second micro-batch
        assert _same_bits(after[1][i][0], after[0][i][0])


def test_ops_moe_empty_batch():
    from distributed_training_guide_b200 import ops

    d = DEBUG
    x, gate_w, gate_up, down, _, _ = _moe_inputs(d["E"], d["k"], d["H"], d["I"], 4, seed=15)
    leaves = [t.clone().requires_grad_() for t in (x[:0], gate_w, gate_up, down)]
    n0 = _ext.launch_count()
    y, psum, counts = ops.moe(*leaves, d["k"])
    assert y.shape == (0, d["H"]) and bool((psum == 0).all()) and bool((counts == 0).all())
    grads = torch.autograd.grad((y, psum), leaves, (torch.zeros_like(y), torch.zeros_like(psum)))
    assert grads[0].shape == (0, d["H"])
    assert all(bool((g == 0).all()) for g in grads[1:])
    assert _ext.launch_count() == n0, "an empty batch launched kernels"


# ------------------------------------------------------------------------------------------------------------------
# table entries outside what they index, and refusals
# ------------------------------------------------------------------------------------------------------------------
MARK = 0x4B19   # bf16 10027008: what a read past an operand would bring back
MARK_F = torch.tensor(MARK, dtype=torch.int16).view(BF16).item()


def _collision():
    """A route for T 64 and the arguments of a batch of T 60: at E 8, k 2 both have rows_cap 1152, so every shape
    check passes and the rows of assignments 120..127 name tokens the batch does not have."""
    E, k, H = 8, 2, 256
    assert _C().moe_rows_cap(64, E, k) == _C().moe_rows_cap(60, E, k) == 1152
    r = _route(torch.randn(64, E, device="cuda", generator=_gen(21)).to(BF16), k)
    return r, E, k, H


def _inside_marks(rows, cols, dtype=BF16, seed=0, after=8, before=8):
    """A [rows, cols] tensor inside a buffer whose ``before`` rows in front of it and ``after`` rows behind it hold
    marks (MARK bits, or 12345.0 in fp32): every row an out-of-range entry could name lies in the buffer, and a read
    of one shows up as a mark."""
    n, b0 = rows * cols, before * cols
    size = (before + rows + after) * cols
    if dtype == BF16:
        buf = torch.full((size,), MARK, device="cuda", dtype=torch.int16).view(BF16)
        buf[b0:b0 + n] = torch.randn(n, device="cuda", generator=_gen(seed)).to(BF16)
    else:
        buf = torch.full((size,), 12345.0, device="cuda", dtype=dtype)
        buf[b0:b0 + n] = torch.rand(n, device="cuda", generator=_gen(seed), dtype=dtype)
    return buf, buf[b0:b0 + n].view(rows, cols)


def test_out_of_range_rows_permute():
    r, E, k, H = _collision()
    T = 60
    buf, x = _inside_marks(T, H)
    before = buf.clone()
    xp = _C().moe_permute(x, r.row_tok, r.seg, k)
    assert _same_bits(buf, before)
    used = r.segs[-1]
    rt = r.row_tok[:used].long()
    bad = rt >= T * k
    good = (rt >= 0) & ~bad
    assert int(bad.sum()) == 8
    marks = int((_bits(xp[:used][bad]) == MARK).all(-1).sum())
    assert bool(torch.isnan(xp[:used][bad]).all()), f"{marks} of 8 rows are mark rows read from past x"
    assert _same_bits(xp[:used][good], x[rt[good] // k])
    assert bool((_bits(xp[:used][rt == -1]) == 0).all())
    # a wrong k with the same rows_cap: k 1 at T 64 has rows_cap 1152 too, and names rows up to 127
    buf64, x64 = _inside_marks(64, H, seed=22, after=64)
    before64 = buf64.clone()
    xp1 = _C().moe_permute(x64, r.row_tok, r.seg, 1)
    assert _same_bits(buf64, before64)
    rt_bad = rt >= 64
    assert bool(torch.isnan(xp1[:used][rt_bad]).all())
    ok = (rt >= 0) & ~rt_bad
    assert _same_bits(xp1[:used][ok], x64[rt[ok]])


def test_out_of_range_rows_combine_backward():
    r, E, k, H = _collision()
    T = 60
    dbuf, dy = _inside_marks(T, H, seed=1)
    wbuf, w = _inside_marks(T, k, dtype=torch.float32, seed=2)
    yp = torch.randn(r.R, H, device="cuda", generator=_gen(3)).to(BF16)
    before = (dbuf.clone(), wbuf.clone())
    dyp, dw = _C().moe_combine_bwd(dy, yp, r.row_tok, r.seg, w)
    assert _same_bits(dbuf, before[0]) and _same_bits(wbuf, before[1])
    used = r.segs[-1]
    rt = r.row_tok[:used].long()
    bad = rt >= T * k
    good = (rt >= 0) & ~bad
    assert bool(torch.isnan(dyp[:used][bad]).all()), \
        f"rows past dy / w were read: {dyp[:used][bad][:, 0].tolist()} (marks: 12345 * {MARK_F})"
    want = (w.reshape(-1)[rt[good], None] * dy[rt[good] // k].float()).to(BF16)
    assert _same_bits(dyp[:used][good], want)
    # every assignment of the batch has a row in the T 64 route, so every dw entry is written, and only those
    ref = (dy.double()[:, None, :] * yp.double()[r.pos[:T].long()]).sum(-1)
    mag = (dy.double().abs()[:, None, :] * yp.double().abs()[r.pos[:T].long()]).sum(-1)
    assert bool(((dw.double() - ref).abs() <= 24 * 2.0 ** -24 * mag).all())


def test_out_of_range_pos_combine():
    C = _C()
    T, k, H = 50, 2, 136
    rows = 256
    buf, yp = _inside_marks(rows, H, seed=4)
    before = buf.clone()
    pos = torch.randint(0, rows, (T, k), device="cuda", generator=_gen(5), dtype=torch.int32)
    pos[3, 1] = rows            # one past yp
    pos[9, 0] = rows + 7        # the last mark row
    pos[20, 1] = -1            # the mark row in front of yp
    w = torch.rand(T, k, device="cuda", generator=_gen(6))
    for wt in (w, None):
        y = C.moe_combine(yp, pos, wt)
        assert _same_bits(buf, before)
        bad = torch.zeros(T, dtype=torch.bool, device="cuda")
        bad[[3, 9, 20]] = True
        assert bool(torch.isnan(y[bad]).all()), f"rows past yp were read: {y[bad][:, 0].tolist()} (mark {MARK_F})"
        wd = wt.double() if wt is not None else torch.ones(T, k, device="cuda", dtype=torch.float64)
        ok = ~bad
        terms = wd[ok][:, :, None] * yp.double()[pos[ok].long()]
        ref = terms.sum(1)
        assert bool(torch.isfinite(y[ok]).all())
        assert bool(((y[ok].double() - ref).abs() <= U * ref.abs() + k * 2.0 ** -24 * terms.abs().sum(1)).all())


def test_refusals_on_wrong_device_or_layout():
    C = _C()
    lg = torch.randn(64, 8, device="cuda").to(BF16)
    p, idx, w, pos, seg, tiles, row_tok, counts = C.moe_route(lg, 2)
    x = torch.randn(64, 256, device="cuda").to(BF16)
    xp = C.moe_permute(x, row_tok, seg, 2)
    R = xp.shape[0]
    W = torch.zeros(8, 256, 256, device="cuda", dtype=BF16)
    out = torch.empty(R, 256, device="cuda", dtype=BF16)

    def strided(t):   # the same values, not contiguous
        return torch.stack([t, t], -1)[..., 0] if t.dim() == 1 else t.transpose(-1, -2).contiguous().transpose(-1, -2)
    with pytest.raises(RuntimeError, match="bf16 CUDA"):
        C.moe_route(lg.cpu(), 2)
    with pytest.raises(RuntimeError, match="contiguous last dimension"):
        C.moe_route(lg.t().contiguous().t(), 2)
    calls = {
        "moe_permute": (lambda a: C.moe_permute(*a), [x, row_tok, seg, 2]),
        "moe_combine": (lambda a: C.moe_combine(*a), [xp, pos, w]),
        "moe_combine_bwd": (lambda a: C.moe_combine_bwd(*a), [x, xp, row_tok, seg, w]),
        "moe_router_bwd": (lambda a: C.moe_router_bwd(*a), [p, idx, w, torch.zeros(8, device="cuda")]),
        "gemm_grouped fwd": (lambda a: C.gemm_grouped(0, *a), [xp, W, out, seg, tiles]),
        "gemm_grouped wgrad": (lambda a: C.gemm_grouped(2, *a),
                               [xp, xp, torch.empty(8, 256, 256, device="cuda", dtype=BF16), seg]),
    }
    for name, (fn, args) in calls.items():
        fn(args)                                                    # the valid call runs
        for i, t in enumerate(args):
            if not isinstance(t, torch.Tensor):
                continue
            for bad in (t.cpu(), strided(t)):
                if bad.is_cuda and bad.is_contiguous():
                    continue
                a = list(args)
                a[i] = bad
                with pytest.raises(RuntimeError, match="device|contiguous|CUDA"):
                    fn(a)
    with pytest.raises(RuntimeError, match="k must be"):
        C.moe_permute(x, row_tok, seg, 9)
    with pytest.raises(RuntimeError, match="pos must be"):
        C.moe_combine(xp, pos[:, :0].contiguous(), None)
    with pytest.raises(RuntimeError, match="yp has no rows"):
        C.moe_combine(xp[:0], pos, None)
