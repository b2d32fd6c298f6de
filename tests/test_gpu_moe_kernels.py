"""The mixture-of-experts kernels against fp64 on one GPU: routing (exact top-k sets, weights and stable-sort rows,
with ties, with every token on the same experts, with empty experts and T not a multiple of 128), the grouped GEMM's
forward, dgrad and wgrad modes (empty experts zero in overwrite mode and untouched in accumulate mode; padding rows
never reach an output), permute / combine and their backward, run-to-run bit identity, and the refusals."""
import pytest
import torch

from distributed_training_guide_b200 import _ext

pytestmark = pytest.mark.gpu


def _C():
    return _ext.load(required=True)


def _route_ref(logits, k):
    """fp64 softmax and the top-k by probability with ties to the lower expert."""
    p = torch.softmax(logits.double(), -1)
    return p, torch.sort(-p, dim=-1, stable=True).indices[:, :k]


def _check_layout(idx, E, pos, seg, tiles, row_tok, counts):
    """The routing tables of ``moe_route``, exactly, from the experts ``idx`` [T, k] it chose: counts, 128-row padded
    segments, each assignment's row in a stable counting sort, row_tok (-1 on padding rows) and the expert of every
    128-row tile up to rows_cap (-1 past the last segment)."""
    T, k = idx.shape
    flat = idx.reshape(-1).long().cpu()
    counts64 = torch.bincount(flat, minlength=E)
    seg64 = torch.zeros(E + 1, dtype=torch.long)
    seg64[1:] = torch.cumsum((counts64 + 127) // 128 * 128, 0)
    order = torch.sort(flat, stable=True).indices                 # assignments grouped by expert, in (t, slot) order
    first = torch.cumsum(counts64, 0) - counts64                  # index into `order` of each expert's first one
    pos64 = torch.empty(T * k, dtype=torch.long)
    pos64[order] = seg64[flat[order]] + torch.arange(T * k) - first[flat[order]]
    assert torch.equal(counts.cpu().long(), counts64)
    assert torch.equal(seg.cpu().long(), seg64)
    assert torch.equal(pos.cpu().long().reshape(-1), pos64)
    used = int(seg64[-1])
    want = torch.full((used,), -1, dtype=torch.int32)
    want[pos64] = torch.arange(T * k, dtype=torch.int32)
    assert torch.equal(row_tok.cpu()[:used], want)
    r = torch.arange(tiles.numel()) * 128
    exp = torch.searchsorted(seg64[1:], r, right=True)            # the expert whose segment holds row r
    exp[r >= used] = -1
    assert torch.equal(tiles.cpu().long(), exp)


def _check_route(logits, k):
    C = _C()
    p, idx, w, pos, seg, tiles, row_tok, counts = C.moe_route(logits, k)
    p64, idx64 = _route_ref(logits.cpu(), k)
    assert torch.equal(idx.cpu().long(), idx64)
    torch.testing.assert_close(p.cpu().double(), p64, rtol=2e-6, atol=1e-7)
    torch.testing.assert_close(w.cpu().double(), p64.gather(1, idx64), rtol=2e-6, atol=1e-7)
    _check_layout(idx, logits.shape[1], pos, seg, tiles, row_tok, counts)
    return p, idx, w, pos, seg, tiles, row_tok, counts


@pytest.mark.parametrize("T,E,k", [(1, 8, 2), (200, 8, 2), (1000, 64, 8), (4096, 64, 8), (300, 256, 4), (77, 40, 3)])
def test_route_random(T, E, k):
    g = torch.Generator(device="cuda").manual_seed(T + E)
    _check_route(torch.randn(T, E, device="cuda", generator=g).to(torch.bfloat16), k)


def test_route_ties_same_experts_and_empty_experts():
    T, E, k = 333, 16, 4
    _check_route(torch.zeros(T, E, device="cuda", dtype=torch.bfloat16), k)   # all tied: experts 0..3 for everyone
    lg = torch.full((T, E), -4.0, device="cuda")
    lg[:, [3, 7, 9, 12]] = 2.0                                               # 12 experts never chosen
    lg[::2, 7] = 3.0
    _, _, _, _, seg, _, _, counts = _check_route(lg.to(torch.bfloat16), k)
    assert int((counts == 0).sum()) == E - 4


def test_route_is_bit_identical_run_to_run():
    lg = torch.randn(4096, 64, device="cuda").to(torch.bfloat16)
    a, b = _C().moe_route(lg, 8), _C().moe_route(lg, 8)
    used = int(a[4][-1])
    for i, (x, y) in enumerate(zip(a, b)):
        if i == 6:   # row_tok: rows past the last segment are never written
            x, y = x[:used], y[:used]
        assert torch.equal(x, y)


def _setup(T, E, k, H, N, seed=0, empty=()):
    g = torch.Generator(device="cuda").manual_seed(seed)
    lg = torch.randn(T, E, device="cuda", generator=g)
    for e in empty:
        lg[:, e] = -30.0
    route = _C().moe_route(lg.to(torch.bfloat16), k)
    x = torch.randn(T, H, device="cuda", generator=g).to(torch.bfloat16)
    return route, x


def _segments(seg, counts):
    return [(int(seg[e]), int(seg[e]) + int(counts[e])) for e in range(len(counts))]


@pytest.mark.parametrize("T,E,k,H,N", [(300, 8, 2, 256, 256), (1000, 16, 4, 512, 384), (2048, 64, 8, 256, 512)])
def test_grouped_forward_dgrad_wgrad_against_fp64(T, E, k, H, N):
    C = _C()
    (p, idx, w, pos, seg, tiles, row_tok, counts), x = _setup(T, E, k, H, N, empty=(1,))
    xp = C.moe_permute(x, row_tok, seg, k)
    R = xp.shape[0]
    segs = _segments(seg.cpu(), counts.cpu())
    # padding rows of the permuted input are zero, real rows are their token's row
    for e, (a, b) in enumerate(segs):
        assert bool((xp[b:int(seg[e + 1])] == 0).all())
    g = torch.Generator(device="cuda").manual_seed(9)
    W = (torch.randn(E, N, H, device="cuda", generator=g) * 0.05).to(torch.bfloat16)
    out = torch.full((R, N), float("nan"), device="cuda", dtype=torch.bfloat16)
    C.gemm_grouped(0, xp, W, out, seg, tiles)
    Wt = W.transpose(1, 2).contiguous()                     # [E, H, N]: dgrad form of the same product
    out1 = torch.full((R, N), float("nan"), device="cuda", dtype=torch.bfloat16)
    C.gemm_grouped(1, xp, Wt, out1, seg, tiles)
    for e, (a, b) in enumerate(segs):
        ref = xp[a:b].double() @ W[e].double().t()
        mag = xp[a:b].double().abs() @ W[e].double().abs().t()
        for got in (out, out1):
            err = (got[a:b].double() - ref).abs()
            assert bool((err <= 2 ** -8 * ref.abs() + 1e-5 * mag + 1e-30).all()), e
            assert bool((got[b:int(seg[e + 1])] == 0).all())   # padding rows: 0 . W
    # wgrad over each expert's rows: dW_e [N, H] = dy_e^T xp_e; expert 1 has no rows
    dy = (torch.randn(R, N, device="cuda", generator=g)).to(torch.bfloat16)
    for e, (a, b) in enumerate(segs):
        dy[b:int(seg[e + 1])] = 0
    dW = torch.full((E, N, H), float("nan"), device="cuda", dtype=torch.bfloat16)
    C.gemm_grouped(2, dy, xp, dW, seg)
    for e, (a, b) in enumerate(segs):
        ref = dy[a:b].double().t() @ xp[a:b].double()
        mag = dy[a:b].double().abs().t() @ xp[a:b].double().abs()
        err = (dW[e].double() - ref).abs()
        assert bool((err <= 2 ** -8 * ref.abs() + 1e-5 * mag + 1e-30).all()), e
    assert int(counts[1]) == 0 and bool((dW[1] == 0).all()) and not bool(torch.signbit(dW[1].float()).any())
    # accumulate: the empty expert's block is left untouched bit for bit (NaN stays NaN, -0 stays -0)
    acc = torch.randn(E, N, H, device="cuda", generator=g).to(torch.bfloat16)
    acc[1] = float("nan")
    acc[1, 0, 0] = -0.0
    before = acc.clone()
    C.gemm_grouped(2, dy, xp, acc, seg, accumulate=True)
    assert torch.equal(acc[1].view(torch.int16), before[1].view(torch.int16))
    for e, (a, b) in enumerate(segs):
        if e == 1:
            continue
        ref = before[e].double() + dy[a:b].double().t() @ xp[a:b].double()
        mag = before[e].double().abs() + dy[a:b].double().abs().t() @ xp[a:b].double().abs()
        assert bool(((acc[e].double() - ref).abs() <= 2 ** -7 * ref.abs() + 1e-5 * mag + 1e-30).all()), e
    # bit-identical on a repeat
    out2 = torch.empty_like(out)
    C.gemm_grouped(0, xp, W, out2, seg, tiles)
    used = int(seg[-1])
    assert torch.equal(out[:used], out2[:used])


def test_combine_and_backward_against_fp64():
    C = _C()
    T, E, k, H = 517, 16, 4, 256
    (p, idx, w, pos, seg, tiles, row_tok, counts), x = _setup(T, E, k, H, H, seed=3)
    R = row_tok.shape[0]
    yp = torch.randn(R, H, device="cuda").to(torch.bfloat16)
    y = C.moe_combine(yp, pos, w)
    ref = (w.double()[:, :, None] * yp.double()[pos.long()]).sum(1)
    assert bool(((y.double() - ref).abs() <= 2 ** -8 * ref.abs() + 1e-6).all())
    dx = C.moe_combine(yp, pos)
    ref1 = yp.double()[pos.long()].sum(1)
    assert bool(((dx.double() - ref1).abs() <= 2 ** -8 * ref1.abs() + 1e-6).all())
    dy = torch.randn(T, H, device="cuda").to(torch.bfloat16)
    dyp, dw = C.moe_combine_bwd(dy, yp, row_tok, seg, w)
    used = int(seg[-1])
    rt = row_tok[:used].long()
    real = rt >= 0
    want = torch.zeros(used, H, dtype=torch.float64, device="cuda")
    want[real] = w.reshape(-1).double()[rt[real], None] * dy.double()[rt[real] // k]
    assert bool(((dyp[:used].double() - want).abs() <= 2 ** -8 * want.abs()).all())
    assert bool((dyp[:used][~real] == 0).all())
    dw_ref = (dy.double()[:, None, :] * yp.double()[pos.long()]).sum(-1)
    mag = (dy.double().abs()[:, None, :] * yp.double().abs()[pos.long()]).sum(-1)
    assert bool(((dw.double() - dw_ref).abs() <= 1e-5 * mag).all())
    # router backward: dlogits = p * (dp - sum p dp)
    dpsum = torch.randn(E, device="cuda")
    dl = C.moe_router_bwd(p, idx, dw, dpsum)
    dp = dpsum.double()[None].repeat(T, 1)
    dp.scatter_add_(1, idx.long(), dw.double())
    ref2 = p.double() * (dp - (p.double() * dp).sum(-1, keepdim=True))
    assert bool(((dl.double() - ref2).abs() <= 2 ** -8 * ref2.abs() + 1e-5 * (p.double() * dp.abs()).sum(-1, keepdim=True)).all())
    a, b = C.moe_combine_bwd(dy, yp, row_tok, seg, w), C.moe_combine_bwd(dy, yp, row_tok, seg, w)
    assert torch.equal(a[0][:used], b[0][:used]) and torch.equal(a[1], b[1])


def test_bad_arguments_are_refused_before_a_launch():
    C = _C()
    lg = torch.randn(64, 8, device="cuda").to(torch.bfloat16)
    with pytest.raises(RuntimeError, match="k must be"):
        C.moe_route(lg, 9)
    with pytest.raises(RuntimeError, match="E must be"):
        C.moe_route(torch.zeros(4, 300, device="cuda", dtype=torch.bfloat16), 2)
    with pytest.raises(RuntimeError, match="bf16"):
        C.moe_route(lg.float(), 2)
    p, idx, w, pos, seg, tiles, row_tok, counts = C.moe_route(lg, 2)
    x = torch.randn(64, 256, device="cuda").to(torch.bfloat16)
    with pytest.raises(RuntimeError, match="row_tok"):
        C.moe_permute(x, row_tok[:-128], seg, 2)
    with pytest.raises(RuntimeError, match="row_tok must be Int"):
        C.moe_permute(x, row_tok.long(), seg, 2)
    xp = C.moe_permute(x, row_tok, seg, 2)
    R = xp.shape[0]
    W = torch.zeros(8, 256, 256, device="cuda", dtype=torch.bfloat16)
    out = torch.empty(R, 256, device="cuda", dtype=torch.bfloat16)
    with pytest.raises(RuntimeError, match="mode"):
        C.gemm_grouped(3, xp, W, out, seg, tiles)
    with pytest.raises(RuntimeError, match="tile_expert"):
        C.gemm_grouped(0, xp, W, out, seg)
    with pytest.raises(RuntimeError, match="one slab per expert"):
        C.gemm_grouped(0, xp, W[:4], out, seg, tiles)
    with pytest.raises(RuntimeError, match="accumulates"):
        C.gemm_grouped(0, xp, W, out, seg, tiles, True)
    with pytest.raises(RuntimeError, match="K % 64"):
        C.gemm_grouped(1, xp[:, :200].contiguous(), torch.zeros(8, 200, 256, device="cuda", dtype=torch.bfloat16),
                       out, seg, tiles)
    with pytest.raises(RuntimeError, match="M % 128"):
        C.gemm_grouped(2, xp[:, :64].contiguous(), xp, torch.empty(8, 64, 256, device="cuda", dtype=torch.bfloat16),
                       seg)
    with pytest.raises(RuntimeError, match="w must be"):
        C.moe_combine(xp, pos, w[:, :1].contiguous())


def test_route_nan_and_inf_logits_give_valid_experts():
    """A non-finite logit row makes every probability NaN: the row still gets k distinct valid experts (the lowest
    indices), NaN weights, and rows inside the segment table; finite rows route as usual."""
    T, E, k = 200, 64, 8
    lg = torch.randn(T, E, device="cuda")
    lg[3, 5] = float("nan")
    lg[17, 0] = float("inf")
    lg[40, :] = float("-inf")
    lg[41, 9] = float("-inf")   # one -inf alone is finite routing: probability 0
    p, idx, w, pos, seg, tiles, row_tok, counts = _C().moe_route(lg.to(torch.bfloat16), k)
    torch.cuda.synchronize()
    idx_c, w_c = idx.cpu(), w.cpu()
    assert bool(((idx_c >= 0) & (idx_c < E)).all())
    for t in range(T):
        assert len(set(idx_c[t].tolist())) == k, t
    for t in (3, 17, 40):
        assert idx_c[t].tolist() == list(range(k)) and bool(torch.isnan(w_c[t]).all()), t
    assert bool(torch.isfinite(w_c[41]).all()) and 9 not in idx_c[41].tolist()
    good = [t for t in range(T) if t not in (3, 17, 40)]
    ref_idx = _route_ref(lg.to(torch.bfloat16)[good].cpu(), k)[1]
    assert torch.equal(idx_c[good].long(), ref_idx)
    used = int(seg[-1])
    assert int(counts.sum()) == T * k and bool((pos >= 0).all()) and bool((pos < used).all())


@pytest.mark.parametrize("H", [8, 136, 384, 896])
def test_combine_backward_at_hidden_sizes_off_the_warp_multiple(H):
    C = _C()
    T, E, k = 150, 8, 2
    (p, idx, w, pos, seg, tiles, row_tok, counts), _ = _setup(T, E, k, H, H, seed=H)
    R = row_tok.shape[0]
    yp = torch.randn(R, H, device="cuda").to(torch.bfloat16)
    dy = torch.randn(T, H, device="cuda").to(torch.bfloat16)
    _, dw = C.moe_combine_bwd(dy, yp, row_tok, seg, w)
    ref = (dy.double()[:, None, :] * yp.double()[pos.long()]).sum(-1)
    mag = (dy.double().abs()[:, None, :] * yp.double().abs()[pos.long()]).sum(-1)
    assert bool(((dw.double() - ref).abs() <= 1e-5 * mag + 1e-30).all())
    y = C.moe_combine(yp, pos, w)
    ref_y = (w.double()[:, :, None] * yp.double()[pos.long()]).sum(1)
    assert bool(((y.double() - ref_y).abs() <= 2 ** -8 * ref_y.abs() + 1e-6).all())
