"""The data-parallel collective kernels (``csrc/comm.cu``, ``csrc/grad_clip.cu``) on one GPU, with 1, 2, 4 and 8 ranks
emulated, against a bit-exact emulation of what the kernels document and against fp64.

Ranks are emulated as in ``test_gpu_dist_gemm_reference.py``: every rank's replica, optimizer shard, signal pad and
slot is a separate guarded tensor on the same device, their ``data_ptr()`` values form the peer-pointer lists, and the
ranks' calls run in rank order on one stream.  Rank r's reduce reads and writes only slice r of the bucket and the
all-gathers only read, so running the ranks one after another computes what the ranks compute together.
``clip_finalize`` reads the other ranks' slots after its barrier: it runs twice over the ranks, and the second pass
reads every slot as the first pass left it.  One GPU cannot test memory ordering between GPUs; the ``multigpu`` tests
stay the check over real NVLink.

Contracts:
- ``allreduce_scale``, ``reduce_scatter`` and the stored values of ``reduce_sumsq``: slice r is bit-identical to an fp32
  sum starting at +0 in the rotated rank order r, r + 1, ..., r - 1, times fp32(scale), rounded once to bf16 (a NaN
  matches any NaN: the kernels' bf16 NaN is not torch's).  Against the fp64 value s·S it is within
  2^-8 |s·S| + (1 + 2^-7) ((NR - 1) 2^-24 s Σ|x_k| + 2^-23 |s·S|) + 2^-133: the bf16 rounding, the fp32 sum, the
  product and fp32(scale) roundings, and half the bf16 subnormal spacing.
- ``rs_adamw`` feeds AdamW the unrounded fp32 sum in the same order.  Each step is held to ``ref.adamw_step`` on that
  sum, on what the kernel read: one bf16 ulp for bf16 values, 1e-6 of the operands for fp32 moments.
- The all-gathers copy bits.  ``reduce_sumsq``'s partials sum, within 2e-6, to the fp64 sum of squares of the stored
  values inside the parameter ranges; ``clip_finalize`` gives every rank the same (norm, coef), with coef equal to
  ``ref.clip_coefficient``; ``adamw_clip`` is held to ``ref.adamw_step(..., coef=coef)`` and writes the same bits to
  every destination.

Every replica sits in a NaN-filled guarded allocation: bytes outside the bucket and slices a call must not write keep
their bits, and padding a call must not use holds NaN.  The kernels spin on signal pads for about 10 s before they
give up and set ``err``.  No call here can reach that: before each launch the test asserts, with the kernel's own
rule ``(int32)(pad - epoch) >= 0``, that every wait the call makes (the exit barrier at epoch + 1 included) is already
satisfied.  After each call ``err`` is still 0 and every pad holds exactly what the protocol wrote: the calling rank's
epoch of its last barrier on channels below ``blocks`` in every rank's pad, and nothing else.
"""
import math
import time

import pytest
import torch

from distributed_training_guide_b200 import _ext
from distributed_training_guide_b200.ops import reference as ref
from test_gpu_dist_gemm_reference import _Guarded, _bits, _pads, _same
from test_gpu_kernels_reference import _refused
from test_gpu_step_reference import _bf16_spacing, _f32

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16
F32 = torch.float32
NAN = float("nan")
U = 2.0 ** -24
MASK32 = 0xFFFFFFFF
LR, B1, B2, EPS = 1e-2, 0.9, 0.999, 1e-8
BF16_MAX = torch.finfo(BF16).max
WRAP = (1 << 32) - 1          # the exit barrier's epoch wraps to 0
HIGH = 3 * (1 << 32) + 7      # SymmGroup's epoch counter is unbounded; the binding keeps the low 32 bits


def _C():
    return _ext.load(True)


def _channels():
    return int(_C().SYMM_MAX_CHANNELS)


@pytest.fixture(scope="module", autouse=True)
def _report_time():
    t0 = time.perf_counter()
    yield
    print(f"\ntest_gpu_comm_reference.py: {time.perf_counter() - t0:.1f} s")


def _guarded(n, dtype=BF16, fill=NAN, seed=99):
    """A ``_Guarded`` view of n elements of any dtype (the guard bits random int32 words)."""
    if dtype == BF16:
        return _Guarded(n, fill=fill, seed=seed)
    g = _Guarded(n * (torch.empty((), dtype=dtype).element_size() // 4), dtype=torch.int32, fill=None, seed=seed)
    g.view = g.view.view(dtype)
    if fill is not None:
        g.view.fill_(fill)
    return g


def _i32(e):
    """The int32 bits of the uint32 epoch e (mod 2^32)."""
    e &= MASK32
    return e - (1 << 32) if e >= 1 << 31 else e


def _agree(got, want):
    """Bit for bit, except that a NaN matches any NaN."""
    return (_bits(got) == _bits(want)) | (torch.isnan(got) & torch.isnan(want))


def _expect(tag, got, want, written):
    """``got`` equals ``want`` bit for bit where ``written`` is False, and agrees with it where True."""
    ok = (_bits(got) == _bits(want)) | (written & torch.isnan(got) & torch.isnan(want))
    bad = int((~ok).sum())
    assert bad == 0, f"{tag}: {bad} elements differ"


def _randn(shape, seed, std=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return std * torch.randn(*shape, device="cuda", generator=g)


def _grads(nr, n, seed):
    """bf16 values over 2^-12 .. 2^12 in magnitude, with some +0 and -0."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(nr, n, device="cuda", generator=g)
    x = x * torch.exp2(torch.randint(-12, 13, (nr, n), device="cuda", generator=g).float())
    u = torch.rand(nr, n, device="cuda", generator=g)
    x = torch.where(u < 0.01, torch.zeros_like(x), x)
    x = torch.where((u >= 0.01) & (u < 0.02), torch.full_like(x, -0.0), x)
    return x.to(BF16)


# ------------------------------------------------------------------------------------------------------------------
# harness
# ------------------------------------------------------------------------------------------------------------------
class _Rig:
    """One guarded signal pad per emulated rank (uint32 [channels][8], random bits until armed), the state every pad
    must hold, and one guarded ``err`` word."""

    def __init__(self, nr, seed):
        self.nr = nr
        self.pads = [_Guarded(_channels() * 8, dtype=torch.int32, fill=None, seed=seed + p) for p in range(nr)]
        self.want = [p.view.clone() for p in self.pads]
        self.err = _Guarded(1, dtype=torch.int32, fill=0, seed=seed + 50)

    def pad_ptrs(self):
        return [p.view.data_ptr() for p in self.pads]

    def arm(self, value, channels):
        """Every rank has already arrived at ``value`` on channels [0, channels)."""
        for p, w in zip(self.pads, self.want):
            p.view.view(-1, 8)[:channels, :self.nr] = _i32(value)
            w.copy_(p.view)

    def assert_cannot_spin(self, r, waits, channels):
        mine = self.pads[r].view.view(-1, 8)[:channels, :self.nr].long() & MASK32
        for e in waits:
            d = (mine - (e & MASK32)) & MASK32
            assert bool((d < (1 << 31)).all()), f"rank {r}'s wait for epoch {e} could spin"

    def run(self, tag, r, epoch, channels, barriers, call, launches=1):
        """Rank r's call, which makes ``barriers`` barriers (at epoch, epoch + 1, ...) on ``channels`` channels."""
        if barriers:
            self.assert_cannot_spin(r, [epoch + k for k in range(barriers)], channels)
        torch.cuda.synchronize()
        n0 = _ext.launch_count()
        call()
        torch.cuda.synchronize()
        assert _ext.launch_count() - n0 == launches, f"{tag}: {_ext.launch_count() - n0} launches, not {launches}"
        assert int(self.err.view.item()) == 0 and self.err.intact(), f"{tag}: a wait timed out"
        if barriers:
            for w in self.want:
                w.view(-1, 8)[:channels, r] = _i32(epoch + barriers - 1)
        for p, (pad, w) in enumerate(zip(self.pads, self.want)):
            assert torch.equal(pad.view, w) and pad.intact(), f"{tag}: signal pad of rank {p}"


class _Replicas:
    """One replica per emulated rank: a bucket of n elements at element ``off`` of a NaN-filled guarded allocation."""

    def __init__(self, nr, n, off, seed, tail=40):
        self.nr, self.n, self.off = nr, n, off
        self.g = [_Guarded(off + n + tail, seed=seed + p) for p in range(nr)]
        self.want = [g.view.clone() for g in self.g]
        self.written = [torch.zeros(g.n, dtype=torch.bool, device="cuda") for g in self.g]

    def bucket(self, p):
        return self.g[p].view[self.off:self.off + self.n]

    def ptrs(self):
        return [g.view.data_ptr() for g in self.g]

    def load(self, data):
        for p in range(self.nr):
            self.bucket(p).copy_(data[p])
            self.want[p].copy_(self.g[p].view)
            self.written[p].zero_()

    def wrote(self, p, lo, vals):
        """Replica p's bucket elements [lo, lo + len(vals)) now hold ``vals``."""
        a = self.off + lo
        self.want[p][a:a + vals.numel()] = vals
        self.written[p][a:a + vals.numel()] = True

    def check(self, tag):
        for p in range(self.nr):
            _expect(f"{tag}: replica {p}", self.g[p].view, self.want[p], self.written[p])
            assert self.g[p].intact(), f"{tag}: wrote outside replica {p}'s allocation"


def _rank_sum(xs, r):
    """fp32 sum of xs[0..NR) from +0 in the rotated order r, r + 1, ..., r - 1."""
    nr = xs.shape[0]
    acc = torch.zeros(xs.shape[1:], device="cuda", dtype=F32)
    for k in range(nr):
        acc = acc + xs[(r + k) % nr].float()
    return acc


def _emulate(xs, r, scale):
    return (_rank_sum(xs, r) * torch.tensor(scale, dtype=F32, device="cuda")).to(BF16)


def _bound_frac(y, xs, scale):
    """Largest fraction of the fp64 bound (module docstring) any finite element of y uses; inf for a miss."""
    nr = xs.shape[0]
    xd = xs.double()
    s = abs(scale)
    sS = xd.sum(0) * scale
    terms = xd.abs().sum(0) * s
    b = 2.0 ** -8 * sS.abs() + (1 + 2.0 ** -7) * ((nr - 1) * U * terms + 2 * U * sS.abs()) + 2.0 ** -133
    yd = y.double()
    fin = torch.isfinite(sS) & torch.isfinite(yd)
    if not bool(fin.any()):
        return 0.0
    return float(((yd - sS).abs() / b)[fin].max())


def _run_reduce(kind, data, per, blocks, elem_off, scale, epoch, seed, ranges=None, tag="", finite=True):
    """Run ``kind`` (allreduce, reduce_scatter, sumsq_bcast or sumsq_rs) for ranks 0..NR-1 over the buckets ``data``
    [NR, NR·per] and check every contract of a reduce; returns what the clipping tests go on with.  ``finite=False``:
    a gradient inside the ranges is NaN or squares past fp32, and the partials are not held to fp64."""
    C = _C()
    nr = data.shape[0]
    n = nr * per
    reps = _Replicas(nr, n, elem_off, seed)
    reps.load(data)
    rig = _Rig(nr, seed + 100)
    rig.arm(epoch + 2, blocks)
    outs = [_Guarded(per, seed=seed + 200 + r) for r in range(nr)] if kind == "reduce_scatter" else None
    sumsq = kind.startswith("sumsq")
    if sumsq:
        table = torch.tensor(ranges, dtype=torch.int64, device="cuda")
        parts = [_guarded(blocks, dtype=torch.float64, fill=NAN, seed=seed + 300 + r) for r in range(nr)]
        inside = torch.zeros(n, dtype=torch.bool, device="cuda")
        for b, e in ranges:
            inside[b:e] = True
    res = {"reps": reps, "rig": rig, "y": [], "frac": 0.0, "sumsq64": [],
           "parts": parts if sumsq else None}
    for r in range(nr):
        sl = slice(r * per, (r + 1) * per)
        xs = data[:, sl]
        y = _emulate(xs, r, scale)
        t = f"{tag} rank {r}"
        if kind == "allreduce":
            def call():
                C.comm_allreduce_scale(reps.ptrs(), rig.pad_ptrs(), elem_off, n, scale, r, epoch, rig.err.view, blocks)
        elif kind == "reduce_scatter":
            def call():
                C.comm_reduce_scatter(reps.ptrs(), outs[r].view, rig.pad_ptrs(), elem_off, n, scale, r, epoch,
                                      rig.err.view, blocks)
        else:
            def call():
                C.comm_reduce_sumsq(reps.ptrs(), rig.pad_ptrs(), elem_off, n, scale, kind == "sumsq_bcast", table,
                                    parts[r].view, r, epoch, rig.err.view, blocks)
        rig.run(t, r, epoch, blocks, 2, call)
        for p in (range(nr) if kind in ("allreduce", "sumsq_bcast") else [r] if kind == "sumsq_rs" else []):
            reps.wrote(p, r * per, y)
        reps.check(t)
        if kind == "reduce_scatter":
            got = outs[r].view
            assert bool(_agree(got, y).all()), f"{t}: out differs from the rotated fp32 sum"
            assert outs[r].intact(), f"{t}: wrote outside out"
        else:
            got = reps.bucket(r)[sl]
        res["y"].append(y)
        res["frac"] = max(res["frac"], _bound_frac(got, xs, scale))
        assert res["frac"] <= 1, f"{t}: fp64 bound fraction {res['frac']:.3g}"
        if sumsq and finite:
            ps = parts[r].view
            assert bool(torch.isfinite(ps).all()) and parts[r].intact(), f"{t}: partials {ps.tolist()}"
            want = float(y.double()[inside[sl]].square().sum())
            got_s = float(ps.sum())
            assert abs(got_s - want) <= 2e-6 * want, f"{t}: partials sum {got_s!r}, fp64 {want!r}"
            res["sumsq64"].append(want)
    return res


# ------------------------------------------------------------------------------------------------------------------
# allreduce_scale and reduce_scatter
# ------------------------------------------------------------------------------------------------------------------
# (blocks, vectors per rank, elem_off): one vector per rank; vector counts that are not a multiple of blocks·512;
# grid-stride loops at 3, 96 (the multi-rank default) and 256 (the one-rank default) blocks; a bucket at a nonzero
# offset inside a larger buffer, as the tensor-parallel norm-gain all-reduce has.
REDUCE_SHAPES = [(1, 1, 0), (1, 1, 296), (3, 1237, 296), (3, 3075, 0), (96, 96 * 512 + 77, 296),
                 (256, 256 * 512 + 5, 0)]


def _scales(nr):
    """(scale, epoch): no scale, the mean, and a loss scale fp32 cannot hold exactly; at a wrapping and a >2^32 epoch."""
    return [(1.0, 5), (1.0 / nr, WRAP), (0.37 / nr, HIGH)]


@pytest.mark.parametrize("kind", ["allreduce", "reduce_scatter"])
@pytest.mark.parametrize("blocks,vecs,elem_off", REDUCE_SHAPES, ids=[f"b{b}-v{v}-off{o}" for b, v, o in REDUCE_SHAPES])
@pytest.mark.parametrize("nr", [1, 2, 4, 8])
def test_reduce_matches_rotated_fp32_sum(nr, blocks, vecs, elem_off, kind):
    per = 8 * vecs
    worst = 0.0
    for i, (scale, epoch) in enumerate(_scales(nr)):
        data = _grads(nr, nr * per, seed=nr * 1000 + vecs + i)
        res = _run_reduce(kind, data, per, blocks, elem_off, scale, epoch, seed=nr + blocks + i,
                          tag=f"{kind} nr{nr} b{blocks} per{per} off{elem_off} scale {scale:.4g} epoch {epoch}")
        worst = max(worst, res["frac"])
    print(f"\n{kind} nr{nr} b{blocks} per{per}: fp64 bound used {worst:.3f}")


def _rotation_data(nr, per):
    """Element j of slice r holds 1, 2^25 and -2^25 on three different ranks (every ordered triple in turn) and 0
    elsewhere.  In fp32 the slice sums to 1 exactly where the 1 comes last of the three in owner r's rotated order."""
    triples = [(a, b, c) for a in range(nr) for b in range(nr) for c in range(nr) if len({a, b, c}) == 3]
    data = torch.zeros(nr, nr * per, dtype=torch.float64)
    for r in range(nr):
        for j in range(per):
            a, b, c = triples[(j + 5 * r) % len(triples)]
            data[a, r * per + j], data[b, r * per + j], data[c, r * per + j] = 1.0, 2.0 ** 25, -2.0 ** 25
    return data.to("cuda").to(BF16)


@pytest.mark.parametrize("kind", ["allreduce", "reduce_scatter", "sumsq_bcast", "sumsq_rs"])
@pytest.mark.parametrize("nr", [4, 8])
def test_reduce_order_is_the_owners_rotation(nr, kind):
    per = 8 * 42      # 336 triples at 8 ranks
    data = _rotation_data(nr, per)
    ranges = [[0, nr * per]]
    res = _run_reduce(kind, data, per, 3, 8, 1.0, 9, seed=nr, ranges=ranges, tag=f"rotation {kind} nr{nr}")
    for r in range(nr):
        y = res["y"][r].float()
        assert bool(((y == 0) | (y == 1)).all()) and 0 < int((y == 1).sum()) < per, f"rank {r}: design not as stated"


def test_reduce_checks_reject_wrong_rotation_and_one_ulp():
    """Self-test: on the designed slices the emulation of a wrong order (every rank starting at rank 0, or at its
    successor) gives different bits than the owner's rotation, and a 1-ulp change of one element is rejected."""
    nr, per = 4, 8 * 42
    data = _rotation_data(nr, per)
    res = _run_reduce("allreduce", data, per, 3, 0, 1.0, 9, seed=3, tag="self-test")
    for r in range(nr):
        xs = data[:, r * per:(r + 1) * per]
        for wrong in ({0} if r else set()) | {(r + 1) % nr}:
            assert not bool(_agree(_emulate(xs, wrong, 1.0), res["y"][r]).all()), f"order from {wrong} not rejected"
    got = res["reps"].bucket(0).clone()
    i = int(got.float().abs().argmax())
    bumped = got.clone()
    bumped[i] = (bumped[i:i + 1].view(torch.int16) + 1).view(BF16)[0]
    with pytest.raises(AssertionError):
        _expect("1 ulp", bumped, got, torch.ones_like(got, dtype=torch.bool))


@pytest.mark.parametrize("kind", ["allreduce", "reduce_scatter"])
@pytest.mark.parametrize("nr", [1, 2, 4, 8])
def test_reduce_special_values_reach_only_their_element(nr, kind):
    """Inf on one rank, +Inf and -Inf on two, NaN on one, and near-bf16-max values whose fp32 sum overflows, or whose
    sum rounds up to Inf in bf16 (bf16 max + half an ulp ties to even, which is Inf), give exactly what the emulation
    gives and leave every other element finite."""
    per = 64
    data = _grads(nr, nr * per, seed=nr + 77).float()
    special = torch.zeros(nr * per, dtype=torch.bool, device="cuda")
    half_ulp = 2.0 ** 119
    for r in range(nr):
        o = r * per
        data[(r + 1) % nr, o + 3] = math.inf
        data[r, o + 17] = NAN
        data[:, o + 24] = BF16_MAX
        data[:, o + 26] = 0.0
        data[0, o + 26] = BF16_MAX
        data[nr - 1, o + 26] = -BF16_MAX if nr > 1 else BF16_MAX
        data[:, o + 27] = 0.0
        data[0, o + 27] = BF16_MAX
        data[nr - 1, o + 27] = half_ulp if nr > 1 else BF16_MAX
        special[[o + 3, o + 17, o + 24, o + 26, o + 27]] = True
        if nr > 1:
            data[0, o + 10], data[nr - 1, o + 10] = math.inf, -math.inf
            special[o + 10] = True
    data = data.to(BF16)
    for scale, epoch in [(1.0, 11), (1.0 / nr, 13)]:
        res = _run_reduce(kind, data, per, 3, 8, scale, epoch, seed=nr, tag=f"special {kind} nr{nr} scale {scale}")
        y = torch.cat(res["y"])
        assert bool(torch.isfinite(y[~special]).all()), "a special value leaked into another element"
        if scale == 1.0 and nr > 1:
            nonfin = (~torch.isfinite(y)).view(nr, per)
            assert bool(nonfin[:, [3, 10, 17, 24, 27]].all()), "designed overflow or non-finite input did not show"


# ------------------------------------------------------------------------------------------------------------------
# rs_adamw: ZeRO-1 (push) and FSDP (param_local)
# ------------------------------------------------------------------------------------------------------------------
def _check_ulp(tag, got, want, operands=None):
    """Every element within one bf16 ulp of want at the magnitude of want or operands (a NaN matches a NaN)."""
    got_f, want_f = got.float(), want.float()
    mag = want_f.abs() if operands is None else torch.maximum(want_f.abs(), operands)
    ulps = (got_f - want_f).abs() / _bf16_spacing(mag)
    ok = (ulps <= 1) | (torch.isnan(got_f) & torch.isnan(want_f))
    assert bool(ok.all()), f"{tag}: {int((~ok).sum())} elements more than 1 bf16 ulp off"


def _check_rel(tag, got, want, scale):
    ok = ((got - want).abs() <= 1e-6 * scale) | (torch.isnan(got) & torch.isnan(want))
    assert bool(ok.all()), f"{tag}: {int((~ok).sum())} elements off by more than 1e-6 of their operands"


def _check_adamw(tag, got, before, g, step, wd, gs, coef=None):
    """One AdamW step of the kernel (p, m, v) from ``before`` on the fp32 gradient ``g`` against ``ref.adamw_step``:
    bf16 values within one ulp, fp32 moments within 1e-6 of their operands (b1·m + (1 - b1)·g may be one FMA)."""
    p, m, v = got
    p0, m0, v0 = before
    pr, mr, vr = p0.clone(), m0.clone(), v0.clone()
    ref.adamw_step(pr, g, mr, vr, _f32(LR), _f32(B1), _f32(B2), _f32(EPS), _f32(wd), step, grad_scale=_f32(gs),
                   coef=coef)
    gc = g.float() * (coef.float() if coef is not None else 1.0) * _f32(gs)
    m_scale = B1 * m0.float().abs() + (1 - B1) * gc.abs()
    if m.dtype == BF16:
        _check_ulp(f"{tag} exp_avg", m, mr, m_scale)
        _check_ulp(f"{tag} exp_avg_sq", v, vr)
    else:
        _check_rel(f"{tag} exp_avg", m, mr, m_scale)
        _check_rel(f"{tag} exp_avg_sq", v, vr, vr.abs())
    _check_ulp(f"{tag} params", p, pr, p0.float().abs())


# (weight decay, first step, grad_scale factor, blocks): decay on and off, a run from step 1 and one in progress at
# step 1000, the mean and a loss scale, one block in grid-stride and the multi-rank default
RS_RUNS = [(0.1, 1, 1.0, 3), (0.0, 1000, 0.37, 96), (0.0, 1, 0.37, 96), (0.1, 1000, 1.0, 3)]


def _rs_adamw_run(nr, push, state, wd, first, gs, blocks, seed, steps=3, drop_rank=None):
    """Runs ``steps`` steps of rs_adamw over nr emulated ranks and checks each rank after its call."""
    C = _C()
    per = 8 * (3 * 512 + 13)
    n, elem_off = nr * per, 40
    grads = _Replicas(nr, n, elem_off, seed)
    rig = _Rig(nr, seed + 100)
    P = (0.05 * _randn((n,), seed + 1)).to(BF16)
    if push:
        params = _Replicas(nr, n, elem_off, seed + 10)
        # replica p holds only slice p: the kernel must read slice r from rank r's replica
        params.load(torch.stack([torch.where((torch.arange(n, device="cuda") // per) == p, P, NAN) for p in range(nr)]))
        local = None
    else:
        local = [_Guarded(per, seed=seed + 20 + r) for r in range(nr)]
        for r in range(nr):
            local[r].view.copy_(P[r * per:(r + 1) * per])
    ms, vs = [], []
    for r in range(nr):
        m = _guarded(per, dtype=state, fill=0.0, seed=seed + 30 + r)
        v = _guarded(per, dtype=state, fill=0.0, seed=seed + 40 + r)
        if first > 1:   # a run in progress: moments of the size the gradients below give
            m.view.copy_(1e-3 * _randn((per,), seed + 50 + r))
            v.view.copy_((1e-2 * _randn((per,), seed + 60 + r)).square())
        ms.append(m)
        vs.append(v)
    hyper = (LR, B1, B2, EPS, wd)
    for step in range(first, first + steps):
        data = (1e-2 * _randn((nr, n), seed + step)).to(BF16)
        grads.load(data)
        epoch = 2 * step + 1
        rig.arm(epoch + 2, blocks)
        for r in range(nr):
            t = f"rs_adamw nr{nr} {'push' if push else 'local'} {state} wd{wd} step {step} rank {r}"
            sl = slice(r * per, (r + 1) * per)
            gsum = _rank_sum(data[:, sl], r)
            p_view = params.bucket(r)[sl] if push else local[r].view
            before = (p_view.clone(), ms[r].view.clone(), vs[r].view.clone())
            others = [(x.view.clone(), x) for q in range(nr) if q != r for x in
                      ([ms[q], vs[q]] + ([] if push else [local[q]]))]

            def call():
                C.comm_rs_adamw(grads.ptrs(), params.ptrs() if push else [], None if push else local[r].view,
                                ms[r].view, vs[r].view, push, rig.pad_ptrs(), elem_off, n, *hyper, step, gs / nr, r,
                                epoch, rig.err.view, blocks)
            rig.run(t, r, epoch, blocks, 2, call)
            grads.check(t)                       # no gradient buffer changes
            new_p = p_view.clone()
            if push:
                for q in range(nr):
                    params.wrote(q, r * per, new_p)
                params.check(t)                  # slice r identical on every replica, nothing else changed
            for snap, x in others:
                assert torch.equal(_bits(x.view), _bits(snap)), f"{t}: another rank's shard changed"
            for x in ms + vs + (local or []):
                assert x.intact(), f"{t}: wrote outside a shard"
            g_check = gsum if drop_rank is None else gsum - data[drop_rank, sl].float()
            _check_adamw(t, (new_p, ms[r].view, vs[r].view), before, g_check, step, wd, gs / nr)


@pytest.mark.parametrize("state", [BF16, F32], ids=["bf16-state", "fp32-state"])
@pytest.mark.parametrize("push", [True, False], ids=["zero1", "fsdp"])
@pytest.mark.parametrize("nr", [1, 2, 4, 8])
def test_rs_adamw_against_reference(nr, push, state):
    for i, (wd, first, gs, blocks) in enumerate(RS_RUNS):
        _rs_adamw_run(nr, push, state, wd, first, gs, blocks, seed=100 * nr + 10 * i + push)


def test_rs_adamw_check_rejects_a_dropped_rank():
    """Self-test: the AdamW check, fed the gradient sum without one rank's part, rejects what the kernel computed."""
    with pytest.raises(AssertionError, match="exp_avg"):
        _rs_adamw_run(4, True, F32, 0.1, 1, 1.0, 3, seed=5, steps=1, drop_rank=2)
    with pytest.raises(AssertionError, match="exp_avg"):
        _rs_adamw_run(2, False, BF16, 0.0, 1000, 0.37, 96, seed=6, steps=1, drop_rank=1)


# ------------------------------------------------------------------------------------------------------------------
# allgather
# ------------------------------------------------------------------------------------------------------------------
# (blocks, shard_off, barrier): on SMs (blocks >= 1, grid-stride at 1 and 3) and on the copy engines (0)
AG_CASES = [(1, 0, True), (3, 88, True), (96, 0, False), (256, 88, False), (0, 0, True), (0, 88, False)]


@pytest.mark.parametrize("nr", [1, 2, 4, 8])
def test_allgather_copies_the_shards_in_rank_order(nr):
    C = _C()
    per = 8 * 1543
    for i, (blocks, shard_off, barrier) in enumerate(AG_CASES):
        shards = _Replicas(nr, per, shard_off, seed=nr + 10 * i)
        data = _randn((nr, per), nr + i).to(BF16)
        shards.load(data)
        rig = _Rig(nr, seed=nr + 10 * i + 5)
        channels = max(blocks, 1)
        rig.arm(9 + 1, channels)
        for r in range(nr):
            full = _Guarded(nr * per + 24, seed=r + 7)
            t = f"allgather nr{nr} blocks {blocks} shard_off {shard_off} {'barrier' if barrier else 'no barrier'} " \
                f"rank {r}"
            rig.run(t, r, 9, channels, 1 if barrier else 0,
                    lambda: C.comm_allgather(shards.ptrs(), full.view, rig.pad_ptrs(), shard_off, per, r, 9,
                                             rig.err.view, barrier, blocks),
                    launches=1 if (blocks > 0 or barrier) else 0)
            assert _same(full.view[:nr * per], data.reshape(-1)), f"{t}: not the shards in rank order"
            assert bool(torch.isnan(full.view[nr * per:].float()).all()) and full.intact(), f"{t}: wrote past NR·per"
            shards.check(t)


# ------------------------------------------------------------------------------------------------------------------
# gradient clipping: reduce_sumsq -> clip_finalize -> adamw_clip
# ------------------------------------------------------------------------------------------------------------------
def _clip_ranges(n):
    """Parameter ranges of a bucket: starting mid-vector, crossing rank-slice boundaries, NaN padding between the
    parameters and at the tail."""
    sizes, gaps = [5003, 17, 8191, 1, 12000, 333, 2900], [5, 8, 13, 3]
    out, b, i = [], 3, 0
    while True:
        e = b + sizes[i % len(sizes)]
        if e > n - 20:
            break
        out.append([b, e])
        b = e + gaps[i % len(gaps)]
        i += 1
    return out


def _clip_data(nr, n, ranges, seed):
    g = (1e-2 * _randn((nr, n), seed)).to(BF16)
    pad = torch.ones(n, dtype=torch.bool, device="cuda")
    for b, e in ranges:
        pad[b:e] = False
    g[:, pad] = NAN
    return g


def _finalize(rig, parts, nr, parity, norm_scale, max_norm, epoch, slots, tag):
    """clip_finalize twice over the ranks with the same parity; returns the second pass's (norm, coef) per rank."""
    C = _C()
    outs = [_guarded(2, dtype=F32, seed=r) for r in range(nr)]
    for pas in range(2):
        rig.arm(epoch + pas + 1, 1)
        for r in range(nr):
            outs[r].view.fill_(NAN)
            rig.run(f"{tag} finalize pass {pas} rank {r}", r, epoch + pas, 1, 1,
                    lambda: C.comm_clip_finalize(parts[r].view, [s.view.data_ptr() for s in slots], rig.pad_ptrs(),
                                                 parity, norm_scale, max_norm, outs[r].view, r, epoch + pas,
                                                 rig.err.view))
    return [o.view.clone() for o in outs]


def _clip_chain(nr, zero1, grads_data, per, blocks, max_norm_rel, states, seed, tag, check_norm=True):
    C = _C()
    n = nr * per
    ranges = _clip_ranges(n)
    gs = 0.37 if zero1 else 0.75
    scale, norm_scale = (gs / nr, 1.0) if zero1 else (1.0 / nr, gs)
    red = _run_reduce("sumsq_rs" if zero1 else "sumsq_bcast", grads_data, per, blocks, 16, scale, WRAP, seed,
                      ranges=ranges, tag=tag, finite=check_norm)
    reps, rig = red["reps"], red["rig"]
    norm64 = math.sqrt(sum(red["sumsq64"])) * norm_scale if check_norm else math.nan
    parity = seed & 1
    slots = [_guarded(2, dtype=torch.float64, seed=seed + r) for r in range(nr)]
    other = [_bits(s.view[1 - parity:2 - parity]).clone() for s in slots]
    max_norm = max_norm_rel * norm64 if math.isfinite(norm64) else 1.0
    outs = _finalize(rig, red["parts"], nr, parity, norm_scale, max_norm, HIGH, slots, tag)
    for r in range(nr):
        assert _same(outs[r], outs[0]), f"{tag}: rank {r}'s (norm, coef) differs from rank 0's"
        assert torch.equal(_bits(slots[r].view[1 - parity:2 - parity]), other[r]) and slots[r].intact(), \
            f"{tag}: the other parity's slot changed"
    norm, coef = outs[0][0:1], outs[0][1:2]
    if check_norm:
        assert abs(float(norm) - norm64) <= 2e-6 * norm64, f"{tag}: norm {float(norm)!r}, fp64 {norm64!r}"
    want = ref.clip_coefficient(norm.cpu(), max_norm).view(1)
    assert torch.equal(coef.cpu(), want) or (math.isnan(float(coef)) and math.isnan(float(want))), \
        f"{tag}: coef {float(coef)!r} for norm {float(norm)!r}, torch gives {float(want)!r}"
    # the update: ZeRO-1 pushes rank r's slice to every replica; plain DDP updates each replica in place
    stored = [reps.bucket(p).clone() for p in range(nr)]
    results = []
    for state in states:
        params = _Replicas(nr, n, 16, seed + 500)
        P = (0.05 * _randn((n,), seed + 501)).to(BF16)
        params.load(P.expand(nr, n))
        size = per if zero1 else n
        ms = [_guarded(size, dtype=state, fill=0.0, seed=seed + 510 + r) for r in range(nr)]
        vs = [_guarded(size, dtype=state, fill=0.0, seed=seed + 520 + r) for r in range(nr)]
        for r in range(nr):
            t = f"{tag} adamw_clip {state} rank {r}"
            lo, hi = (r * per, (r + 1) * per) if zero1 else (0, n)
            src = params.bucket(r)[lo:hi]
            g = stored[r][lo:hi]
            before = (src.clone(), ms[r].view.clone(), vs[r].view.clone())
            if zero1:
                dst = [params.ptrs()[(r + k) % nr] + 2 * (16 + lo) for k in range(nr)]
            else:
                dst = [src.data_ptr()]
            coef_r = outs[r][1:]
            C.comm_adamw_clip(dst, 0, src, g, ms[r].view, vs[r].view, LR, B1, B2, EPS, 0.1, 1,
                              1.0 if zero1 else gs, coef_r)
            torch.cuda.synchronize()
            new = src.clone()
            for q in (range(nr) if zero1 else [r]):
                params.wrote(q, lo, new)
            params.check(t)
            assert ms[r].intact() and vs[r].intact(), f"{t}: wrote outside the optimizer state"
            _check_adamw(t, (new, ms[r].view, vs[r].view), before, g.float(), 1, 0.1, 1.0 if zero1 else gs, coef_r)
            results.append(new)
    return outs[0], results


@pytest.mark.parametrize("mode", ["ddp", "zero1"])
@pytest.mark.parametrize("nr", [1, 2, 4, 8])
def test_clip_chain_against_fp64(nr, mode):
    zero1 = mode == "zero1"
    per = 8 * (3 * 512 * 2 + 5)
    n = nr * per
    for rel, blocks in ((0.3, 3), (1e30, 96)):     # coef < 1, and coef exactly 1
        data = _clip_data(nr, n, _clip_ranges(n), seed=nr + 7 * zero1)
        out, _ = _clip_chain(nr, zero1, data, per, blocks, rel, [BF16, F32], seed=nr * 10 + zero1 + blocks,
                             tag=f"clip {mode} nr{nr} max_norm {rel}·norm")
        assert (float(out[1]) < 1) if rel < 1 else (float(out[1]) == 1.0)


@pytest.mark.parametrize("mode", ["ddp", "zero1"])
@pytest.mark.parametrize("nr", [2, 4])
def test_clip_chain_nan_and_inf(nr, mode):
    """A NaN gradient element gives a NaN norm and coef and a NaN in every updated parameter, as in torch; a finite
    gradient whose square overflows fp32 gives an Inf norm and coef 0."""
    zero1 = mode == "zero1"
    per = 8 * 1600
    n = nr * per
    ranges = _clip_ranges(n)
    data = _clip_data(nr, n, ranges, seed=nr)
    data[1, ranges[1][0]] = NAN
    out, new = _clip_chain(nr, zero1, data, per, 3, 0.5, [F32], seed=nr + 40, tag=f"nan {mode} nr{nr}",
                           check_norm=False)
    assert math.isnan(float(out[0])) and math.isnan(float(out[1]))
    assert all(bool(torch.isnan(p.float()).all()) for p in new), "a parameter survived a NaN coefficient"
    data = _clip_data(nr, n, ranges, seed=nr + 1)
    data[0, ranges[2][0] + 1] = 2.0 ** 70
    out, _ = _clip_chain(nr, zero1, data, per, 3, 0.5, [BF16], seed=nr + 60, tag=f"inf {mode} nr{nr}",
                         check_norm=False)
    assert math.isinf(float(out[0])) and float(out[1]) == 0.0


# ------------------------------------------------------------------------------------------------------------------
# refusals: each raises before any launch.  Operands sit inside guarded allocations.
# ------------------------------------------------------------------------------------------------------------------
CPU = torch.device("cpu")


def _base(nr=2, per=64, off=8):
    reps = _Replicas(nr, nr * per, off, seed=1)
    reps.load(torch.zeros(nr, nr * per, device="cuda", dtype=BF16))
    pads = _pads(nr)
    err = torch.zeros(1, device="cuda", dtype=torch.int32)
    return reps, [p.data_ptr() for p in pads], err, pads


def _bad_common(call, ptrs_name, ptrs, pads, err, offset_name=None, count_name="n"):
    """Refusals every peer-pointer binding shares."""
    _refused(call(**{ptrs_name: ptrs * 5, "pads": pads * 5}), "1..8 ranks")
    _refused(call(pads=pads[:1]), "pads must have 2 entries")
    _refused(call(pads=pads + pads[:1]), "pads must have 2 entries")
    _refused(call(pads=[pads[0], 0]), "every entry of pads must be a 16-byte aligned")
    _refused(call(**{ptrs_name: [ptrs[0], ptrs[1] + 2]}), f"every entry of {ptrs_name} must be a 16-byte aligned")
    _refused(call(rank=2), "rank 2 outside")
    _refused(call(rank=-1), "rank -1 outside")
    if count_name:
        _refused(call(**{count_name: -128}), f"{count_name} must not be negative")
    if offset_name:
        _refused(call(**{offset_name: -8}), f"{offset_name} must be a non-negative multiple of 8")
        _refused(call(**{offset_name: 4}), f"{offset_name} must be a non-negative multiple of 8")
    _refused(call(err=err.to(CPU)), "err must be an int32 tensor")
    _refused(call(err=err.long()), "err must be an int32 tensor")


def test_allreduce_scale_and_reduce_scatter_refusals():
    C = _C()
    reps, pads, err, _keep = _base()
    out = _Guarded(64 + 8)
    base = dict(buf=reps.ptrs(), pads=pads, elem_off=8, n=128, scale=1.0, rank=0, epoch=1, err=err, blocks=3)

    def ar(**kw):
        a = {**base, **kw}
        return lambda: C.comm_allreduce_scale(a["buf"], a["pads"], a["elem_off"], a["n"], a["scale"], a["rank"],
                                              a["epoch"], a["err"], a["blocks"])
    _bad_common(ar, "buf", reps.ptrs(), pads, err, "elem_off")

    def rs(**kw):
        a = {**base, "grads": reps.ptrs(), "out": out.view[:64], **kw}
        return lambda: C.comm_reduce_scatter(a["grads"], a["out"], a["pads"], a["elem_off"], a["n"], a["scale"],
                                             a["rank"], a["epoch"], a["err"], a["blocks"])
    _bad_common(rs, "grads", reps.ptrs(), pads, err, "elem_off")
    _refused(rs(out=out.view[:64].to(CPU)), "out must be on")
    _refused(rs(out=out.view[1:65]), "out must start at a 16-byte aligned")
    _refused(rs(out=out.view[:64].float()), "out must be BFloat16")
    reps.check("refusals")
    assert out.intact()


@pytest.mark.parametrize("push", [True, False], ids=["zero1", "fsdp"])
def test_rs_adamw_refusals(push):
    C = _C()
    reps, pads, err, _keep = _base()
    params, _, _, _ = _base()
    per = 64
    mg, vg, pg = (_guarded(2 * per + 8, dtype=F32, fill=0.0, seed=i) for i in range(3))
    pl = _Guarded(2 * per + 8, fill=0.0, seed=4)
    base = dict(grads=reps.ptrs(), params=params.ptrs() if push else [], param_local=None if push else pl.view[:per],
                m=mg.view[:per], v=vg.view[:per], pads=pads, elem_off=8, n=128, rank=0, err=err)

    def call(**kw):
        a = {**base, **kw}
        return lambda: C.comm_rs_adamw(a["grads"], a["params"], a["param_local"], a["m"], a["v"], push, a["pads"],
                                       a["elem_off"], a["n"], LR, B1, B2, EPS, 0.0, 1, 0.5, a["rank"], 1, a["err"], 3)
    _bad_common(call, "grads", reps.ptrs(), pads, err, "elem_off")
    for name, g in (("m", mg), ("v", vg)):
        _refused(call(**{name: g.view[:per].to(CPU)}), f"{name} must be on")
        _refused(call(**{name: g.view[:2 * per:2]}), f"{name} must be contiguous")
        _refused(call(**{name: g.view[1:per + 1]}), f"{name} must start at a 16-byte aligned")
    if push:
        _refused(call(params=params.ptrs()[:1]), "params must have 2 entries")
        _refused(call(params=[params.ptrs()[0], params.ptrs()[1] + 8]), "every entry of params must be")
    else:
        _refused(call(param_local=pl.view[:per].to(CPU)), "param_local must be on")
        _refused(call(param_local=pl.view[:2 * per:2]), "param_local must be contiguous")
        _refused(call(param_local=pl.view[1:per + 1]), "param_local must start at a 16-byte aligned")
        _refused(call(param_local=pg.view[:per]), "param_local must be BFloat16")
    reps.check("refusals")
    assert all(g.intact() for g in (mg, vg, pg, pl))


def test_allgather_refusals():
    C = _C()
    nr, per = 2, 64
    shards, pads, err, _keep = _base(nr, per, 8)     # each rank's shard: `per` elements at element 8
    full = _Guarded(4 * per + 8, fill=0.0)
    for blocks in (3, 0):
        base = dict(shards=shards.ptrs(), full=full.view[:nr * per], pads=pads, shard_off=8, per=per, rank=0, err=err)

        def ag(**kw):
            a = {**base, **kw}
            return lambda: C.comm_allgather(a["shards"], a["full"], a["pads"], a["shard_off"], a["per"], a["rank"], 1,
                                            a["err"], True, blocks)
        _bad_common(ag, "shards", shards.ptrs(), pads, err, "shard_off", "per")
        _refused(ag(full=full.view[:nr * per].to(CPU)), "full must be on")
        _refused(ag(full=full.view[1:nr * per + 1]), "full must start at a 16-byte aligned")
        _refused(ag(full=full.view[:nr * per].float()), "full must be BFloat16")
        _refused(ag(full=full.view[:nr * per - 8]), "full buffer too small")
    shards.check("refusals")
    assert full.intact() and bool((full.view == 0).all())


def test_clipping_refusals():
    C = _C()
    reps, pads, err, _keep = _base()
    table = torch.tensor([[0, 100]], device="cuda", dtype=torch.int64)
    parts = torch.zeros(3, device="cuda", dtype=torch.float64)
    base = dict(buf=reps.ptrs(), pads=pads, elem_off=8, n=128, rank=0, err=err)

    def ss(**kw):
        a = {**base, **kw}
        return lambda: C.comm_reduce_sumsq(a["buf"], a["pads"], a["elem_off"], a["n"], 0.5, False, table, parts,
                                           a["rank"], 1, a["err"], 3)
    _bad_common(ss, "buf", reps.ptrs(), pads, err, "elem_off")
    slots = [_guarded(2, dtype=torch.float64, seed=s) for s in range(2)]
    out = torch.zeros(2, device="cuda")
    fb = dict(slots=[s.view.data_ptr() for s in slots], pads=pads, rank=0, err=err)

    def fin(**kw):
        a = {**fb, **kw}
        return lambda: C.comm_clip_finalize(parts, a["slots"], a["pads"], 0, 1.0, 1.0, out, a["rank"], 1, a["err"])
    _refused(fin(rank=2), "rank 2 outside")
    _refused(fin(rank=-1), "rank -1 outside")
    _refused(fin(slots=[fb["slots"][0], fb["slots"][1] + 8]), "every entry of slots must be")
    _refused(fin(pads=[pads[0], 0]), "every entry of pads must be")
    _refused(fin(err=err.to(CPU)), "err must be an int32 tensor")
    n = 64
    p = _Guarded(n, fill=1.0, seed=1)
    g = _Guarded(n, fill=1.0, seed=2)
    mg, vg = _guarded(2 * n + 8, dtype=F32, fill=0.0, seed=3), _guarded(2 * n + 8, dtype=F32, fill=0.0, seed=4)
    coef = torch.ones(1, device="cuda")
    ab = dict(dst=[p.view.data_ptr()], m=mg.view[:n], v=vg.view[:n])

    def ac(**kw):
        a = {**ab, **kw}
        return lambda: C.comm_adamw_clip(a["dst"], 0, p.view, g.view, a["m"], a["v"], LR, B1, B2, EPS, 0.0, 1, 1.0,
                                         coef)
    for name, t in (("m", mg), ("v", vg)):
        _refused(ac(**{name: t.view[:n].to(CPU)}), f"{name} must be on")
        _refused(ac(**{name: t.view[:2 * n:2]}), f"{name} must be contiguous")
        _refused(ac(**{name: t.view[1:n + 1]}), f"{name} must start at a 16-byte aligned")
    _refused(ac(dst=[p.view.data_ptr() + 2]), "every entry of dst must be")
    _refused(lambda: C.comm_barrier(pads, 2, 1, err), "rank 2 outside")
    reps.check("refusals")
    assert all(t.intact() for t in (p, g, mg, vg) + tuple(slots))
