"""The bias epilogue of the wgmma GEMM and the bias-gradient kernel.

Bias epilogue: ``out = bf16(acc + b)`` (fp8: ``bf16(acc * deq + b)``) must be bit-identical to the same kernel run in
accumulate mode over a C prefilled with the broadcast bias, which adds a bf16 C to the fp32 accumulators with the
same operation order.  That holds for the 1-CTA and the CTA-pair variants, for the fp8 forward GEMM, for the FSDP
gather GEMM (register epilogue) and for the all-gather GEMM, at ragged M and N.  Against fp64 the result is within
one bf16 rounding of ``acc + b`` (plus the fp32 accumulation error), also where ``b`` cancels ``acc``.  A NaN or Inf
bias entry reaches exactly its column; repeated calls are bit-identical; every binding refusal happens before a
launch.

Bias gradient: fp32 column sums of a bf16 [T, N] against fp64, bit-identical from run to run, and routed into a flat
gradient view with overwrite-then-accumulate."""
import pytest
import torch

from distributed_training_guide_b200 import _ext, ops

pytestmark = pytest.mark.gpu

MS = (1, 127, 4097)
NS = (1152, 4608, 8, 264)


def _C():
    return _ext.load()


def _operands(M, N, K, seed, bias_scale=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = (torch.randn(M, K, device="cuda", generator=g) * 0.5).to(torch.bfloat16)
    w = (torch.randn(N, K, device="cuda", generator=g) * 0.05).to(torch.bfloat16)
    b = (torch.randn(N, device="cuda", generator=g) * bias_scale).to(torch.bfloat16)
    return x, w, b


def _prefilled(b, M):
    return b[None, :].expand(M, -1).contiguous()


@pytest.mark.parametrize("variant", [1, 2])
@pytest.mark.parametrize("M", MS)
@pytest.mark.parametrize("N", NS)
def test_bias_epilogue_matches_accumulate_over_prefilled_bias(variant, M, N):
    C = _C()
    x, w, b = _operands(M, N, 320, seed=M * 7 + N)
    out = torch.full((M, N), float("nan"), device="cuda", dtype=torch.bfloat16)
    C.gemm(x, w, out, False, True, False, variant, bias=b)
    want = _prefilled(b, M)
    C.gemm(x, w, want, False, True, True, variant)
    assert torch.equal(out, want), (out.float() - want.float()).abs().max()


def test_bias_epilogue_at_qwen25_7b_qkv_shape():
    C = _C()
    x, w, b = _operands(4096, 4608, 3584, seed=1)
    for variant in (1, 2):
        out = torch.empty(4096, 4608, device="cuda", dtype=torch.bfloat16)
        C.gemm(x, w, out, False, True, False, variant, bias=b)
        want = _prefilled(b, 4096)
        C.gemm(x, w, want, False, True, True, variant)
        assert torch.equal(out, want)


def _fp8_operands(M, N, K, seed):
    x, w, b = _operands(M, N, K, seed)
    x8, _, sx = ops.fp8_cast(x, torch.float8_e4m3fn, transposed=False)
    w8, _, sw = ops.fp8_cast(w, torch.float8_e4m3fn, transposed=False)
    return x8, sx, w8, sw, b


@pytest.mark.parametrize("variant", [1, 2])
@pytest.mark.parametrize("M", MS)
@pytest.mark.parametrize("N", (1152, 4608, 16, 272))
def test_fp8_bias_epilogue_matches_accumulate_over_prefilled_bias(variant, M, N):
    C = _C()
    x8, sx, w8, sw, b = _fp8_operands(M, N, 256, seed=M + 3 * N)
    out = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
    C.gemm_fp8(x8, w8, out, sx, sw, False, variant, bias=b)
    want = _prefilled(b, M)
    C.gemm_fp8(x8, w8, want, sx, sw, True, variant)
    assert torch.equal(out, want), (out.float() - want.float()).abs().max()


def _single_rank_symm():
    from distributed_training_guide_b200.parallel.symm import SymmGroup

    return SymmGroup(torch.device("cuda", torch.cuda.current_device()), ranks=[0])


def test_gather_gemm_bias_matches_accumulate_over_prefilled_bias():
    """B_MODE 3 (FSDP unshard inside the GEMM, register epilogue) on one rank: the whole weight is the local shard."""
    sg = _single_rank_symm()
    C = sg.C
    shift = 15
    M, N, K = 4097, 1152, 512
    x, w, b = _operands(M, N, K, seed=5)
    n = N * K
    shard = sg.alloc(n, torch.bfloat16)
    shard.local.copy_(w.reshape(-1))
    full = shard.local.clone()
    counters = torch.zeros(max(64, (n * 2) >> shift), device="cuda", dtype=torch.int32)
    out = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
    C.gemm_bgather(x, full, out, True, N, K, shard.ptrs, n, 0, n, counters, 2, shift, sg.pad_ptrs, 0, 0, b)
    want = _prefilled(b, M)
    C.gemm(x, w, want, False, True, True, 2)
    torch.cuda.synchronize()
    assert torch.equal(out, want), (out.float() - want.float()).abs().max()
    with pytest.raises(RuntimeError, match="bias"):
        C.gemm_bgather(x[:, :N].contiguous(), full, torch.empty(M, K, device="cuda", dtype=torch.bfloat16), False, N,
                       K, shard.ptrs, n, 0, n, counters, 2, shift, sg.pad_ptrs, 0, 0, b)


def test_all_gather_gemm_bias_matches_accumulate_over_prefilled_bias():
    """A_MODE 3 (tensor parallelism's all-gather GEMM) on one rank."""
    sg = _single_rank_symm()
    C = sg.C
    M, N, K = 512, 1152, 256
    x, w, b = _operands(M, N, K, seed=9)
    a = sg.alloc(M * K, torch.bfloat16)
    a.local.copy_(x.reshape(-1))
    flags = torch.zeros(max(1, M // 256), device="cuda", dtype=torch.int32)
    out = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
    C.gemm_ag(a.ptrs, w, out, True, 0, M, flags, 1, sg.pad_ptrs, sg._epochs(1), 4, b)
    want = _prefilled(b, M)
    C.gemm(x, w, want, False, True, True, 2)
    torch.cuda.synchronize()
    assert torch.equal(out, want), (out.float() - want.float()).abs().max()
    with pytest.raises(RuntimeError, match="bias"):
        C.gemm_ag(a.ptrs, w.t().contiguous(), out, False, 0, M, flags, 2, sg.pad_ptrs, sg._epochs(1), 4, b)


def _within_one_rounding(out, x, w, b):
    """|out - (x w^T + b)| <= half a bf16 ulp of the exact value, plus the fp32 accumulation error."""
    exact = x.double() @ w.double().t() + b.double()
    absdot = x.double().abs() @ w.double().abs().t()
    K = x.shape[1]
    bound = exact.abs() * 2.0 ** -8 + absdot * K * 2.0 ** -23 + 1e-30
    err = (out.double() - exact).abs()
    assert bool((err <= bound).all()), (err / bound).max()


@pytest.mark.parametrize("variant", [1, 2])
@pytest.mark.parametrize("M,N", [(127, 264), (4097, 1152), (1, 8)])
def test_bias_epilogue_against_fp64(variant, M, N):
    C = _C()
    x, w, b = _operands(M, N, 640, seed=11 + M, bias_scale=4.0)
    out = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
    C.gemm(x, w, out, False, True, False, variant, bias=b)
    _within_one_rounding(out, x, w, b)


@pytest.mark.parametrize("variant", [1, 2])
def test_bias_epilogue_cancellation(variant):
    """b = -bf16(acc) for row 0: the output of row 0 is what is left of acc after the cancellation, rounded once."""
    C = _C()
    M, N, K = 256, 1152, 896
    x, w, _ = _operands(M, N, K, seed=21)
    acc = x[:1].double() @ w.double().t()
    b = (-acc[0]).to(torch.bfloat16)
    out = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
    C.gemm(x, w, out, False, True, False, variant, bias=b)
    _within_one_rounding(out, x, w, b)
    assert float(out[0].float().abs().max()) < float(acc.abs().max()) * 2.0 ** -6


def test_nonfinite_bias_reaches_exactly_its_column():
    C = _C()
    M, N, K = 300, 1152, 256
    x, w, b = _operands(M, N, K, seed=31)
    for bad, col in ((float("nan"), 5), (float("inf"), 700), (float("-inf"), 1151)):
        bb = b.clone()
        bb[col] = bad
        out = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
        C.gemm(x, w, out, False, True, False, 2, bias=bb)
        others = torch.cat([out[:, :col], out[:, col + 1:]], dim=1)
        assert bool(torch.isfinite(others).all())
        if bad != bad:
            assert bool(out[:, col].isnan().all())
        else:
            assert bool((out[:, col].float() == bad).all())


def test_repeated_calls_are_bit_identical():
    C = _C()
    x, w, b = _operands(4097, 4608, 896, seed=41)
    outs = []
    for _ in range(3):
        out = torch.empty(4097, 4608, device="cuda", dtype=torch.bfloat16)
        C.gemm(x, w, out, False, True, False, 0, bias=b)
        outs.append(out)
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2])


def test_gemm_bias_refusals():
    C = _C()
    M, N, K = 128, 264, 64
    x, w, b = _operands(M, N, K, seed=51)
    out = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
    sentinel = torch.full_like(out, 7.0)
    bad = {
        "bfloat16": b.float(),
        "contiguous": torch.empty(2 * N, device="cuda", dtype=torch.bfloat16)[::2],
        r"\[N\]": torch.zeros(N + 8, device="cuda", dtype=torch.bfloat16),
        "device": b.cpu(),
        "16-byte": torch.zeros(N + 1, device="cuda", dtype=torch.bfloat16)[1:],
    }
    for msg, bb in bad.items():
        out.copy_(sentinel)
        with pytest.raises(RuntimeError, match=msg):
            C.gemm(x, w, out, False, True, False, 0, bias=bb)
        assert torch.equal(out, sentinel), msg
    with pytest.raises(RuntimeError, match="accumulate"):
        C.gemm(x, w, out, False, True, True, 0, bias=b)
    with pytest.raises(RuntimeError, match="forward layout"):
        C.gemm(x.t().contiguous(), w, out, True, True, False, 0, bias=b)
    with pytest.raises(RuntimeError, match="forward layout"):
        C.gemm(x, w.t().contiguous(), out, False, False, False, 0, bias=b)
    assert torch.equal(out, sentinel)
    x8, sx, w8, sw, b16 = _fp8_operands(M, 272, K, seed=52)
    o8 = torch.empty(M, 272, device="cuda", dtype=torch.bfloat16)
    with pytest.raises(RuntimeError, match="accumulate"):
        C.gemm_fp8(x8, w8, o8, sx, sw, True, 0, bias=b16)
    with pytest.raises(RuntimeError, match="bfloat16"):
        C.gemm_fp8(x8, w8, o8, sx, sw, False, 0, bias=b16.float())
    with pytest.raises(RuntimeError, match="e4m3"):
        C.gemm_fp8(x8.view(torch.float8_e5m2), w8, o8, sx, sw, False, 0, bias=b16)


# ---------------------------------------------------------------------------------------------------------------
# bias gradient
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("T", (1, 127, 4097))
@pytest.mark.parametrize("N", (8, 264, 1152, 4608))
def test_bias_grad_against_fp64_and_bit_identical(T, N):
    C = _C()
    g = torch.Generator(device="cuda").manual_seed(T + N)
    dy = (torch.randn(T, N, device="cuda", generator=g) * 3).to(torch.bfloat16)
    db = C.bias_grad(dy)
    assert db.dtype == torch.float32 and db.shape == (N,)
    exact = dy.double().sum(0)
    bound = dy.double().abs().sum(0) * T * 2.0 ** -24 + 1e-30
    assert bool(((db.double() - exact).abs() <= bound).all())
    if T == 1:
        assert torch.equal(db, dy[0].float())
    assert torch.equal(db, C.bias_grad(dy))


def test_bias_grad_row_stride_and_refusals():
    C = _C()
    big = torch.randn(300, 1160, device="cuda").to(torch.bfloat16)
    view = big[:, :1152]   # row stride 1160
    assert torch.equal(C.bias_grad(view), C.bias_grad(view.contiguous()))
    for msg, bad in (("bfloat16", view.float()), ("2-D", big[None]), ("contiguous last", big.t()),
                     ("multiple of 8", big[:, :12].contiguous())):
        with pytest.raises(RuntimeError, match=msg):
            C.bias_grad(bad)


def test_bias_grad_overwrites_then_accumulates_into_a_flat_view():
    from distributed_training_guide_b200.models.llama import FusedWeight

    flat_p = torch.zeros(2048, device="cuda", dtype=torch.bfloat16)
    flat_g = torch.full((2048,), 123.0, device="cuda", dtype=torch.bfloat16)   # never zeroed: stale values
    owner = FusedWeight(flat_p[8:8 + 1152], flat_g[8:8 + 1152])
    dy1 = torch.randn(500, 1152, device="cuda").to(torch.bfloat16)
    dy2 = torch.randn(700, 1152, device="cuda").to(torch.bfloat16)
    assert ops._emit_bias_grad(owner, dy1, owner.data) is None
    first = ops.bias_grad(dy1).to(torch.bfloat16)
    assert torch.equal(flat_g[8:8 + 1152], first)
    ops._emit_bias_grad(owner, dy2, owner.data)
    assert torch.equal(flat_g[8:8 + 1152], first + ops.bias_grad(dy2).to(torch.bfloat16))
    assert bool((flat_g[:8] == 123.0).all()) and bool((flat_g[8 + 1152:] == 123.0).all())


def test_linear_with_bias_through_autograd():
    x = torch.randn(4, 64, 256, device="cuda").to(torch.bfloat16).requires_grad_()
    w = (torch.randn(1152, 256, device="cuda") * 0.05).to(torch.bfloat16).requires_grad_()
    b = torch.randn(1152, device="cuda").to(torch.bfloat16).requires_grad_()
    y = ops.linear(x, w, b)
    want = ops.gemm(x.detach().reshape(-1, 256), w.detach(), trans_b=True, bias=b.detach())
    assert torch.equal(y.reshape(-1, 1152), want)
    dy = torch.randn_like(y)
    y.backward(dy)
    assert torch.equal(b.grad, ops.bias_grad(dy.reshape(-1, 1152)).to(torch.bfloat16))
    xr, wr, br = x.detach().float().requires_grad_(), w.detach().float().requires_grad_(), b.detach().float()
    br.requires_grad_()
    torch.nn.functional.linear(xr, wr, br).backward(dy.float())
    for got, want in ((x.grad, xr.grad), (w.grad, wr.grad), (b.grad, br.grad)):
        assert ((got.float() - want).norm() / want.norm()).item() < 1e-2
