"""The kernels indexed by token id or vocabulary column against fp64, on one GPU: the cross-entropy loss, the
vocabulary-parallel loss, and the embedding forward and backward, plain and hidden-parallel (tensor-parallel).

The tensor-parallel kernels run here by emulating the shards: every rank's shard, stats and gradient buffers are
separate tensors on the same device, their ``data_ptr()`` values form the peer-pointer list, and the ranks' calls run in
rank order on one stream.  The volatile stats loads of ``vp_ce_grad`` and the pulls of ``tp_embed_*`` are valid on local
addresses, so no second GPU or symmetric memory is needed.

Cross-entropy bound, every element, no outlier budget.  With p64 = exp(x - lse64) the fp64 softmax of the same bf16
logits, d64 = (p64 - onehot) / n_valid and

    eps = 2^-24 (C0 + C1 |x - lse64| + C2 V/512 + |lse64|),

each dlogit must satisfy |d - d64| <= 2^-8 |d64| + (p64 eps + 2^-126) / n_valid + 2^-134.
- 2^-8 |d64|: the final bf16 rounding (half an ulp is at most 2^-8 of the value).
- |x - lse| and |lse|: the fp32 subtraction x - lse and the rounding of lse = max + log(sum) (one 2^-24 each).
- C1 = 4: __expf is within 2 + floor(1.173 |y|) ulp (2^-23 each), so (4 + 2.35 |y|) 2^-24 relative, plus the
  subtraction's 2^-24 |y|.
- C2 = 2: each thread adds V/512 exponentials in fp32 (V/8 vectors of 8 over 512 threads), one rounding of at most 2^-24
  of the row sum each; doubled for the rescales of the online max.
- C0 = 128: __logf's 3 ulp on log(sum) <= log(V) < 12 (48), the pass-1 __expf errors weighted by the softmax, whose
  mean |y| is at most log V (32), the 9-level block reduction (9), the reciprocal and the product (2), rounded up.
- 2^-126: __expf flushes a result below fp32's smallest normal to zero; 2^-134: bf16 subnormal rounding.
A dlogit moved by 2 bf16 ulps, a row's lse off by 2^-12, or a target one column off exceeds the bound (self-test).
The loss must be within the mean over valid rows of 2^-24 (C0 + C2 V/512 + |lse64| + |l64|) plus the fp32 sum of T row
losses, 2^-24 (ceil(T/1024) + 10) sum |l64| / n_valid, plus the division's 2^-24 |loss64|.

Embedding backward rows follow the rule of ``test_embedding_backward_rows_against_fp64``: at most 1.5x the error of the
correctly rounded row.  The forward is bit-identical to ``w[ids]``.

Out-of-vocabulary ids and targets (tests named ``*out_of_vocab*``) come only from {-101, -2, -1, V, V + 1}, and the
logits, tables and gradients they could reach are views inside sentinel rows, so that even a kernel that dereferenced
them stays inside the test's own buffers.
"""
import math

import pytest
import torch

from distributed_training_guide_b200 import _ext, ops
from test_gpu_kernels_reference import EMB_FACTOR, EMB_SLACK, _gen, _ids, _refused, _row_rel
from test_gpu_step_reference import _bf16_spacing

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16
IGNORE = -100
C0, C1, C2 = 128.0, 4.0, 2.0
U = 2.0 ** -24
BAD_IDS = (-101, -2, -1)   # and V, V + 1
PAD_BEFORE, PAD_AFTER = 104, 2   # rows around a table: -101 stays inside
SENTINEL = 7.0

# every vocabulary the model registry trains, and small and ragged ones (4104: 513 vectors, one thread takes two)
REGISTRY_V = [32000, 49152, 50304, 50432, 50688, 100352, 128256, 151936, 152064]
CE_CASES = [(V, T) for V in [8, 16, 4096, 4104] + REGISTRY_V for T in (1, 7, 1024)] + [(151936, 4096), (152064, 4096)]


def _C():
    return _ext.load(True)


def _bits(t):
    return t.contiguous().view(torch.int16)


# ------------------------------------------------------------------------------------------------------------------
# inputs and the fp64 reference
# ------------------------------------------------------------------------------------------------------------------
DESIGNS = ("randn", "randn4", "peaked", "at_min", "equal", "neg_inf", "edge")


def _ce_inputs(T, V, seed, ignore="random", cols=None):
    """bf16 logits [T, V] and int64 targets.  Row i has design DESIGNS[(i + seed) % 7]: randn x 1 and x 4; the target
    25 above the rest (p - 1 cancels); the target at the row's minimum; all logits equal; 1 % of entries -inf; targets
    cycling through ``cols`` (default: columns 0, V - 1 and the last 16-byte vector, which a ragged row gives to one
    thread as an extra)."""
    g = _gen(seed)
    x = torch.randn(T, V, device="cuda", generator=g)
    design = (torch.arange(T, device="cuda") + seed) % len(DESIGNS)
    tgt = torch.randint(0, V, (T,), device="cuda", generator=g)

    def rows(name):
        return (design == DESIGNS.index(name)).nonzero().squeeze(1)

    x[rows("randn4")] *= 4
    r = rows("equal")
    x[r] = x[r, :1]
    r = rows("at_min")
    x[r] *= 2
    tgt[r] = x[r].argmin(1)
    r = rows("peaked")
    x[r, tgt[r]] = x[r].max(1).values + 25
    r = rows("neg_inf")
    x[r] = (2 * x[r]).masked_fill(torch.rand(len(r), V, device="cuda", generator=g) < 0.01, -math.inf)
    x[r, tgt[r]] = 0.0
    r = rows("edge")
    cols = cols if cols is not None else [0, V - 1] + list(range(max(V - 8, 0), V - 1))
    tgt[r] = torch.tensor(cols, device="cuda")[torch.arange(len(r), device="cuda") % len(cols)]
    if ignore == "random" and T > 1:
        tgt[torch.rand(T, device="cuda", generator=g) < 1 / 7] = IGNORE
    elif ignore == "ends":
        tgt[0] = tgt[-1] = IGNORE
    elif ignore == "all_but_one":
        tgt[torch.arange(T, device="cuda") != T // 2] = IGNORE
    return x.to(BF16), tgt


def _ce_fracs(d, loss, x, tgt):
    """Largest fraction of the bound (module docstring) that any dlogit and the loss use; inf for a NaN, or for a
    nonzero dlogit of an ignored row."""
    T, V = x.shape
    valid = tgt != IGNORE
    nv = max(int(valid.sum()), 1)
    worst, at = 0.0, None
    lsum = labs = lterm = 0.0
    for r0 in range(0, T, 256):
        r1 = min(T, r0 + 256)
        xs, ts, vs = x[r0:r1].double(), tgt[r0:r1], valid[r0:r1]
        lse = torch.logsumexp(xs, 1)
        p = torch.exp(xs - lse[:, None])
        rows = vs.nonzero().squeeze(1)
        oh = torch.zeros_like(p)
        oh[rows, ts[rows]] = 1
        vsd = vs.double()[:, None]
        d64 = (p - oh) * vsd / nv
        eps = U * (C0 + C1 * (xs - lse[:, None]).abs() + C2 * V / 512 + lse.abs()[:, None])
        pe = torch.where(p > 0, p * eps, torch.zeros_like(p))
        bound = (2.0 ** -8 * d64.abs() + (pe + 2.0 ** -126) / nv + 2.0 ** -134) * vsd
        err = (d[r0:r1].double() - d64).abs()
        frac = torch.where(bound > 0, err / bound.clamp_min(1e-300), torch.where(err == 0, 0.0, math.inf))
        frac = torch.where(torch.isnan(frac), math.inf, frac)
        m = frac.max()
        if m.item() > worst:
            worst = m.item()
            i = int(frac.argmax())
            at = (r0 + i // V, i % V)
        l64 = lse[rows] - xs[rows, ts[rows]]
        lsum += l64.sum().item()
        labs += l64.abs().sum().item()
        lterm += (U * (C0 + C2 * V / 512 + lse[rows].abs() + l64.abs())).sum().item()
    loss64 = lsum / nv
    lbound = lterm / nv + U * (math.ceil(T / 1024) + 10) * labs / nv + U * abs(loss64)
    lerr = abs(float(loss) - loss64)
    lfrac = lerr / lbound if lbound > 0 else (0.0 if lerr == 0 else math.inf)
    if math.isnan(lfrac):
        lfrac = math.inf
    return worst, at, lfrac


def _ce_run(x, tgt):
    y = x.clone()
    loss = _C().cross_entropy_fwd_bwd(y, tgt)
    return y, loss


def _check_ce(tag, d, loss, x, tgt):
    fd, at, fl = _ce_fracs(d, loss, x, tgt)
    print(f"\n{tag}: worst dlogit at {at}: {fd:.3g} of its bound; loss {fl:.3g} of its bound")
    assert fd <= 1, f"{tag}: dlogit at (row, column) {at} uses {fd:.3g} of its bound"
    assert fl <= 1, f"{tag}: loss uses {fl:.3g} of its bound"
    ign = (tgt == IGNORE).nonzero().squeeze(1)
    assert int(torch.count_nonzero(_bits(d[ign]))) == 0, f"{tag}: an ignored row is not bit-zero"


# ------------------------------------------------------------------------------------------------------------------
# cross-entropy
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("V,T", CE_CASES)
def test_cross_entropy_against_fp64(V, T):
    x, tgt = _ce_inputs(T, V, seed=V % 7)
    d, loss = _ce_run(x, tgt)
    d2, loss2 = _ce_run(x, tgt)
    assert torch.equal(_bits(d), _bits(d2)) and torch.equal(loss.view(torch.int32), loss2.view(torch.int32)), \
        "a second call gave other bits"
    _check_ce(f"V {V} T {T}", d, loss, x, tgt)


@pytest.mark.parametrize("ignore", ["ends", "all_but_one"])
@pytest.mark.parametrize("T", [7, 1024])
@pytest.mark.parametrize("V", [8, 4104, 32000, 152064])
def test_cross_entropy_ignored_rows_against_fp64(V, T, ignore):
    x, tgt = _ce_inputs(T, V, seed=3, ignore=ignore)
    d, loss = _ce_run(x, tgt)
    _check_ce(f"V {V} T {T} {ignore}", d, loss, x, tgt)


@pytest.mark.parametrize("V", [8, 4104, 152064])
def test_cross_entropy_near_bf16_max_against_fp64(V):
    """Rows with entries at +-bf16 max beside randn ones (the target at the largest), and rows whose every logit lies
    just above -bf16 max: no overflow to inf or NaN, and the fp64 bound, whose |lse| term covers the rounding of lse."""
    T, top = 7, 3.3895e38
    g = _gen(11)
    x = torch.randn(T, V, device="cuda", generator=g)
    tgt = torch.randint(0, V, (T,), device="cuda", generator=g)
    for r in range(5):
        c = torch.randperm(V, device="cuda", generator=g)[:4]
        x[r, c] = torch.tensor([top, 0.99 * top, -top, -0.99 * top], device="cuda")
        tgt[r] = c[0]
    x[5:] = -top * (1 - 0.01 * torch.rand(2, V, device="cuda", generator=g))
    x = x.to(BF16)
    assert torch.isfinite(x).all()
    d, loss = _ce_run(x, tgt)
    assert torch.isfinite(d).all() and torch.isfinite(loss)
    _check_ce(f"near bf16 max V {V}", d, loss, x, tgt)


def test_cross_entropy_bound_rejects_small_errors():
    """The bound of this file rejects each of: one dlogit moved by 2 bf16 ulps, a row's lse off by 2^-12 (on a peaked
    row, where p - 1 cancels), a target one column off."""
    V, T = 32000, 64
    x, tgt = _ce_inputs(T, V, seed=0, ignore="none")
    d, loss = _ce_run(x, tgt)
    assert _ce_fracs(d, loss, x, tgt)[0] <= 1
    nv = T
    r = DESIGNS.index("peaked")            # seed 0: row r has that design
    xs = x[r].double()
    lse = torch.logsumexp(xs, 0)

    def row(shift=0.0, t=None):
        t = int(tgt[r]) if t is None else t
        p = torch.exp(xs - lse - shift)
        p[t] -= 1
        return (p / nv).to(BF16)

    moved = d.clone()
    c = int(d[0].float().abs().argmax())
    moved.view(torch.int16)[0, c] += 2
    lse_off = d.clone()
    lse_off[r] = row(shift=2.0 ** -12)
    col_off = d.clone()
    col_off[r] = row(t=(int(tgt[r]) + 1) % V)
    for name, bad in (("2 ulps", moved), ("lse + 2^-12", lse_off), ("target + 1", col_off)):
        f = _ce_fracs(bad, loss, x, tgt)[0]
        print(f"\n{name}: {f:.3g} of the bound")
        assert f > 1, f"the bound accepts {name}"


@pytest.mark.parametrize("V", [4104, 128256])
def test_cross_entropy_upstream_gradient(V):
    """Through ``ops.cross_entropy``: an upstream gradient of 0.5 gives exactly half the kernel's bits, 1/3 stays within
    two roundings of the kernel's dlogits / 3."""
    T = 256
    x, tgt = _ce_inputs(T, V, seed=5)
    d, _ = _ce_run(x, tgt)
    for s in (0.5, 1 / 3):
        xl = x.clone().requires_grad_(True)
        (ops.cross_entropy(xl.clone(), tgt) * s).backward()
        if s == 0.5:
            assert torch.equal(_bits(xl.grad), _bits((d.float() * 0.5).to(BF16))), "0.5 x dlogits is not exact"
        else:
            want = d.double() / 3
            err = (xl.grad.double() - want).abs()
            assert bool((err <= _bf16_spacing(want.float()).double()).all()), f"1/3: worst {err.max():.3g}"


def test_cross_entropy_nan_logit_poisons_its_row_only():
    V, T, r = 32000, 64, 5
    x, tgt = _ce_inputs(T, V, seed=2, ignore="none")
    xn = x.clone()
    xn[r, 100] = math.nan
    d, loss = _ce_run(x, tgt)
    dn, lossn = _ce_run(xn, tgt)
    assert torch.isnan(dn[r]).all(), "the NaN row's dlogits are not all NaN"
    assert torch.isnan(lossn), "the loss is not NaN"
    others = torch.arange(T, device="cuda") != r
    assert torch.equal(_bits(dn[others]), _bits(d[others])), "a NaN changed other rows"


# ------------------------------------------------------------------------------------------------------------------
# vocabulary-parallel cross-entropy, N shards emulated on one GPU
# ------------------------------------------------------------------------------------------------------------------
def _vp_run(x, tgt, N, pad=0):
    """Every rank's stats, then every rank's gradient, in rank order.  Returns the concatenated dlogits, each rank's
    loss and the shards (views ``pad`` rows inside their own buffers)."""
    C = _C()
    T, V = x.shape
    Vl = V // N
    bufs, shards = [], []
    for k in range(N):
        b = torch.full((T + 2 * pad, Vl), SENTINEL, device="cuda", dtype=BF16)
        b[pad:pad + T] = x[:, k * Vl:(k + 1) * Vl]
        bufs.append(b)
        shards.append(b[pad:pad + T])
    stats = [torch.empty(4 * T, device="cuda") for _ in range(N)]
    for k in range(N):
        C.vp_ce_stats(shards[k], tgt, stats[k], k * Vl)
    ptrs = [s.data_ptr() for s in stats]
    losses = [C.vp_ce_grad(shards[k], tgt, ptrs, k * Vl) for k in range(N)]
    return torch.cat(shards, 1), losses, bufs


@pytest.mark.parametrize("N", [1, 2, 4, 8])
@pytest.mark.parametrize("V", [2048, 32000, 128256, 151936])
def test_vocab_parallel_cross_entropy_against_fp64(V, N):
    """Every rank returns the same loss bits; the concatenated dlogits and the loss meet the cross-entropy bound, with
    targets at the shard edges k Vl - 1 and k Vl.  With one shard the kernels are the plain loss bit for bit: the
    reductions are the same, the single combine factor is __expf(0) = 1 exactly, and 1 x the target logit is exact."""
    T, Vl = 512, V // N
    cols = sorted({0, V - 1} | {k * Vl + e for k in range(1, N) for e in (-1, 0)})
    x, tgt = _ce_inputs(T, V, seed=N, cols=cols)
    d, losses, _ = _vp_run(x, tgt, N)
    bits = {int(l.view(torch.int32)) for l in losses}
    assert len(bits) == 1, f"ranks returned different losses: {[float(l) for l in losses]}"
    if N == 1:
        dp, lp = _ce_run(x, tgt)
        assert torch.equal(_bits(d), _bits(dp)) and torch.equal(losses[0].view(torch.int32), lp.view(torch.int32)), \
            "one shard differs from the plain loss"
    _check_ce(f"vocab-parallel V {V} N {N}", d, losses[0], x, tgt)


# ------------------------------------------------------------------------------------------------------------------
# embedding forward, plain and hidden-parallel
# ------------------------------------------------------------------------------------------------------------------
def _padded_table(V, H, fill):
    """A [V, H] view with PAD_BEFORE sentinel rows before it and PAD_AFTER after, and its buffer."""
    b = torch.full((PAD_BEFORE + V + PAD_AFTER, H), SENTINEL, device="cuda", dtype=BF16)
    b[PAD_BEFORE:PAD_BEFORE + V] = fill
    return b, b[PAD_BEFORE:PAD_BEFORE + V]


def _sentinels_intact(b, V):
    return bool((b[:PAD_BEFORE] == SENTINEL).all() and (b[PAD_BEFORE + V:] == SENTINEL).all())


def _tp_embed_fwd(ids, w, N):
    """Rank k looks up columns [k Hl, (k + 1) Hl) of every token and stores them into the owner's [rpp, H] buffer.
    Returns the [T, H] result and the ranks' padded table buffers."""
    C = _C()
    T, (V, H) = ids.numel(), w.shape
    Hl, rpp = H // N, -(-T // N)
    tables = [_padded_table(V, Hl, w[:, k * Hl:(k + 1) * Hl]) for k in range(N)]
    dst = [torch.empty(rpp, H, device="cuda", dtype=BF16) for _ in range(N)]
    ptrs = [t.data_ptr() for t in dst]
    for k in range(N):
        C.tp_embed_fwd(ids, tables[k][1], ptrs, rpp, H, k)
    return torch.cat(dst, 0)[:T], [b for b, _ in tables]


@pytest.mark.parametrize("N", [0, 2, 4, 8])
def test_embedding_forward_bit_exact(N):
    """N = 0: the plain kernel.  T x H / 8 vectors (4M) exceed both launchers' grid caps, so the grid-stride loops run."""
    V, H, T = 32000, 4096, 8192
    g = _gen(21)
    w = torch.randn(V, H, device="cuda", generator=g).to(BF16)
    ids = torch.randint(0, V, (T,), device="cuda", generator=g)
    ids[:2] = torch.tensor([0, V - 1], device="cuda")
    out = _C().embedding_fwd(ids, w) if N == 0 else _tp_embed_fwd(ids, w, N)[0]
    assert torch.equal(_bits(out), _bits(w[ids]))


# ------------------------------------------------------------------------------------------------------------------
# hidden-parallel embedding backward
# ------------------------------------------------------------------------------------------------------------------
def _tp_embed_bwd(ids, dx, dws, accumulate):
    """Rank k pulls its columns of every token's dx row from the owner (rank t / rpp) and sums them into dws[k]."""
    C = _C()
    N = len(dws)
    T, H = dx.shape
    rpp = -(-T // N)
    parts = [torch.zeros(rpp, H, device="cuda", dtype=BF16) for _ in range(N)]
    for k in range(N):
        parts[k][:min(rpp, T - k * rpp)] = dx[k * rpp:(k + 1) * rpp]
    ptrs = [p.data_ptr() for p in parts]
    for k in range(N):
        C.tp_embed_bwd(ids, ptrs, dws[k], rpp, H, k, accumulate)
    return torch.cat(dws, 1)


def _rows_vs_exact(tag, got, exact, present):
    rel = _row_rel(got[present], exact[present])
    rel_cr = _row_rel(exact[present].to(BF16), exact[present])
    ratio = rel / rel_cr.clamp_min(1e-30)
    print(f"\n{tag}: worst row {ratio.max().item():.2f}x the correctly rounded error")
    bad = rel > EMB_FACTOR * rel_cr + EMB_SLACK
    assert not bad.any(), f"{tag}: {int(bad.sum())} rows beyond {EMB_FACTOR}x the correctly rounded error " \
                          f"(worst {ratio.max().item():.2f}x)"


@pytest.mark.parametrize("kind,T,N", [("zipf1.0", 4096, 2), ("zipf1.2", 4096, 2), ("zipf1.0", 16384, 2),
                                      ("pad", 4096, 2), ("uniform", 4096, 2), ("zipf1.0", 4096, 8)])
def test_tp_embedding_backward_rows_against_fp64(kind, T, N):
    """Overwrite over a table holding last step's values (absent rows come out zero), then accumulate a second batch:
    every row within 1.5x the error of the correctly rounded row."""
    V, H = 32000, 4096
    Hl = H // N
    ids = _ids(kind, T, V)
    dx1 = (1e-3 * torch.randn(T, H, device="cuda", generator=_gen(1))).to(BF16)
    dx2 = (1e-3 * torch.randn(T, H, device="cuda", generator=_gen(2))).to(BF16)
    dws = [torch.randn(V, Hl, device="cuda", generator=_gen(3 + k)).to(BF16) for k in range(N)]
    got = _tp_embed_bwd(ids, dx1, dws, False)
    exact = torch.zeros(V, H, device="cuda", dtype=torch.float64).index_add_(0, ids, dx1.double())
    present = torch.bincount(ids, minlength=V) > 0
    assert int(torch.count_nonzero(got[~present])) == 0, "overwrite left rows of absent ids nonzero"
    _rows_vs_exact(f"{kind} T {T} N {N} overwrite", got, exact, present)
    got2 = _tp_embed_bwd(ids, dx2, dws, True)
    exact2 = got.double().index_add_(0, ids, dx2.double())
    assert torch.equal(got2[~present], got[~present]), "accumulate changed rows of absent ids"
    _rows_vs_exact(f"{kind} T {T} N {N} accumulate", got2, exact2, present)


# ------------------------------------------------------------------------------------------------------------------
# out-of-vocabulary ids and targets
# ------------------------------------------------------------------------------------------------------------------
def _bad_values(V):
    return list(BAD_IDS) + [V, V + 1]


def test_cross_entropy_out_of_vocab_targets():
    """A target outside [0, V) other than -100: counted in n_valid, NaN row loss (so NaN loss), NaN dlogits row; every
    other row exactly as with that target made valid.  Rows before and after the logits stay untouched."""
    V, T = 4104, 16
    x, tgt = _ce_inputs(T, V, seed=4, ignore="none")
    tgt[3] = IGNORE
    bad_rows = [0, 5, 8, 11, T - 1]
    for r, b in zip(bad_rows, _bad_values(V)):
        tgt[r] = b
    buf = torch.full((T + 4, V), SENTINEL, device="cuda", dtype=BF16)
    buf[2:T + 2] = x
    loss = _C().cross_entropy_fwd_bwd(buf[2:T + 2], tgt)
    assert torch.isnan(loss), "the mean loss is not NaN"
    assert bool((buf[:2] == SENTINEL).all() and (buf[T + 2:] == SENTINEL).all()), "a sentinel row changed"
    d = buf[2:T + 2]
    bad = torch.zeros(T, dtype=torch.bool, device="cuda")
    bad[bad_rows] = True
    assert torch.isnan(d[bad]).all(), "a bad target's row is not all NaN"
    assert not torch.isnan(d[~bad]).any(), "NaN outside the bad rows"
    fixed = tgt.clone()
    fixed[bad] = 0
    dv, _ = _ce_run(x, fixed)
    assert torch.equal(_bits(d[~bad]), _bits(dv[~bad])), "a bad target changed other rows"


@pytest.mark.parametrize("N", [2, 8])
def test_vocab_parallel_cross_entropy_out_of_vocab_targets(N):
    V, T = 2048, 16
    x, tgt = _ce_inputs(T, V, seed=6, ignore="none")
    bad_rows = [1, 4, 9, 12, T - 1]
    for r, b in zip(bad_rows, _bad_values(V)):
        tgt[r] = b
    d, losses, bufs = _vp_run(x, tgt, N, pad=2)
    assert all(torch.isnan(l) for l in losses), "a rank's loss is not NaN"
    for b in bufs:
        assert bool((b[:2] == SENTINEL).all() and (b[T + 2:] == SENTINEL).all()), "a sentinel row changed"
    bad = torch.zeros(T, dtype=torch.bool, device="cuda")
    bad[bad_rows] = True
    assert torch.isnan(d[bad]).all() and not torch.isnan(d[~bad]).any(), "NaN rows not exactly at the bad targets"
    fixed = tgt.clone()
    fixed[bad] = 0
    dv, _, _ = _vp_run(x, fixed, N)
    assert torch.equal(_bits(d[~bad]), _bits(dv[~bad])), "a bad target changed other rows"


def _oov_ids(T, V, seed):
    g = _gen(seed)
    ids = torch.randint(0, 40, (T,), device="cuda", generator=g)       # repeated ids
    bad = torch.randperm(T, device="cuda", generator=g)[:T // 4]
    vals = torch.tensor(_bad_values(V), device="cuda")
    ids[bad] = vals[torch.arange(len(bad), device="cuda") % len(vals)]
    return ids, ids >= 0


@pytest.mark.parametrize("N", [0, 2])
def test_embedding_forward_out_of_vocab_ids(N):
    """N = 0: the plain kernel.  A bad id's row is NaN, every other row is w[id]; the table's sentinels stay."""
    V, H, T = 1000, 256, 512
    w = torch.randn(V, H, device="cuda", generator=_gen(7)).to(BF16)
    ids, _ = _oov_ids(T, V, 8)
    ok = (ids >= 0) & (ids < V)
    if N == 0:
        b, wv = _padded_table(V, H, w)
        out, bufs = _C().embedding_fwd(ids, wv), [b]
    else:
        out, bufs = _tp_embed_fwd(ids, w, N)
    assert all(_sentinels_intact(b, V) for b in bufs), "a sentinel row around the table changed"
    assert torch.isnan(out[~ok]).all(), "a bad id's row is not all NaN"
    assert torch.equal(_bits(out[ok]), _bits(w[ids[ok]]))


@pytest.mark.parametrize("path", ["default", "sorted", "tp"])
@pytest.mark.parametrize("accumulate", [False, True])
def test_embedding_backward_out_of_vocab_ids(path, accumulate):
    """Bad ids add to no row: the table equals the one from the same batch without them, bit for bit (the gradients
    are multiples of 2^-6 whose sums are exact in fp32, so the order of the atomics cannot show), and the sentinel
    rows around dw stay.  V = 1000: 4V mod 512 = 416, so the slot table's allocation has room past its end."""
    V, H, T = 1000, 256, 2048
    ids, _ = _oov_ids(T, V, 9)
    ok = (ids >= 0) & (ids < V)
    dout = (torch.randint(-64, 64, (T, H), device="cuda", generator=_gen(10)).float() * 2.0 ** -6).to(BF16)
    old = torch.randn(V, H, device="cuda", generator=_gen(12)).to(BF16)
    C = _C()

    N = 2 if path == "tp" else 1      # the tp path: each rank's [V, H / 2] shard inside its own sentinel rows
    Hl = H // N

    def run(i, g):
        tables = [_padded_table(V, Hl, old[:, k * Hl:(k + 1) * Hl]) for k in range(N)]
        dws = [dw for _, dw in tables]
        if path == "default":
            C.embedding_bwd(g, i, dws[0], accumulate)
        elif path == "sorted":
            if not accumulate:
                dws[0].zero_()
            srt, perm = torch.sort(i, stable=True)
            C.embedding_bwd_sorted(g, srt.contiguous(), perm.contiguous(), dws[0], True)
        else:
            _tp_embed_bwd(i, g, dws, accumulate)
        assert all(_sentinels_intact(b, V) for b, _ in tables), "a sentinel row around dw changed"
        return torch.cat(dws, 1)

    got = run(ids, dout)
    want = run(ids[ok].contiguous(), dout[ok].contiguous())
    assert torch.equal(_bits(got), _bits(want)), "bad ids changed the table"


# ------------------------------------------------------------------------------------------------------------------
# argument checks: refused before any launch; no rows, no launch
# ------------------------------------------------------------------------------------------------------------------
def test_loss_and_embedding_bindings_refuse_bad_arguments():
    C = _C()
    T, V, H = 64, 256, 128
    dev = "cuda"
    bf = lambda *s: torch.zeros(*s, device=dev, dtype=BF16)           # noqa: E731
    tgt = torch.zeros(T, device=dev, dtype=torch.long)
    x = bf(T, V)
    for f in (lambda lg, t: C.cross_entropy_fwd_bwd(lg, t),
              lambda lg, t: C.vp_ce_stats(lg, t, torch.zeros(4 * T, device=dev), 0),
              lambda lg, t: C.vp_ce_grad(lg, t, [torch.zeros(4 * T, device=dev).data_ptr()], 0)):
        _refused(lambda: f(bf(2, T // 2, V), tgt), "2-D")
        _refused(lambda: f(bf(T, 12), tgt), "multiple of 8")
        _refused(lambda: f(x, tgt.int()), "int64")
        _refused(lambda: f(x, torch.zeros(2 * T, device=dev, dtype=torch.long)[::2]), "contiguous")
        _refused(lambda: f(x, tgt.cpu()), "device")
        _refused(lambda: f(x, tgt[:-1]), "one entry per logits row")
    st = torch.zeros(4 * T + 4, device=dev)
    _refused(lambda: C.vp_ce_stats(x, tgt, st.double(), 0), "fp32")
    _refused(lambda: C.vp_ce_stats(x, tgt, st[1:], 0), "16-byte")
    _refused(lambda: C.vp_ce_stats(x, tgt, st[:4 * T - 4], 0), "4 floats per row")
    _refused(lambda: C.vp_ce_stats(x, tgt, st, 8), "v0")
    p = st.data_ptr()
    _refused(lambda: C.vp_ce_grad(x, tgt, [p + 4], 0), "16-byte")
    _refused(lambda: C.vp_ce_grad(x, tgt, [p, p], 8), "v0")
    _refused(lambda: C.vp_ce_grad(x, tgt, [p, p], 2 * V), "v0")
    _refused(lambda: C.vp_ce_grad(x, tgt, [p, p, p], 0), "1, 2, 4 or 8")

    ids = torch.zeros(T, device=dev, dtype=torch.long)
    N, rpp = 2, T // 2
    dst = [bf(rpp, H).data_ptr() for _ in range(N)]
    w = bf(V, H // N)
    for f in (lambda i, t, ptrs, r, k: C.tp_embed_fwd(i, t, ptrs, r, H, k),
              lambda i, t, ptrs, r, k: C.tp_embed_bwd(i, ptrs, t, r, H, k, False)):
        _refused(lambda: f(ids.int(), w, dst, rpp, 0), "int64")
        _refused(lambda: f(ids.cpu(), w, dst, rpp, 0), "device")
        _refused(lambda: f(ids, w.float(), dst, rpp, 0), "wrong dtype")
        _refused(lambda: f(ids, torch.zeros(V * H // N + 8, device=dev, dtype=BF16)[1:1 + V * H // N].view(V, H // N),
                           dst, rpp, 0), "must start")
        _refused(lambda: f(ids, bf(V, 36), dst, rpp, 0), "multiple of 8")
        _refused(lambda: f(ids, w, dst, rpp, N), "outside")
        _refused(lambda: f(ids, w, dst, rpp, -1), "outside")
        _refused(lambda: f(ids, w, dst, rpp - 1, 0), "do not fit")

    # no rows: no launch, and the loss of an empty batch is 0 (as with every target ignored)
    torch.cuda.synchronize()
    n0 = _ext.launch_count()
    e = torch.zeros(0, device=dev, dtype=torch.long)
    assert float(C.cross_entropy_fwd_bwd(bf(0, V), e)) == 0.0
    C.vp_ce_stats(bf(0, V), e, torch.zeros(4, device=dev), 0)
    assert float(C.vp_ce_grad(bf(0, V), e, [p], 0)) == 0.0
    assert C.embedding_fwd(e, bf(V, H)).shape == (0, H)
    C.tp_embed_fwd(e, w, dst, rpp, H, 0)
    torch.cuda.synchronize()
    assert _ext.launch_count() == n0, "a call with no rows launched a kernel"
