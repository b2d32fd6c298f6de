"""The renormalised routing of Qwen3-MoE (``norm_topk_prob``) against fp64 on one GPU, and the grouped GEMM at
Qwen3-MoE's shapes.

Bounds and contracts, none with an outlier budget:

- Route with ``norm_topk``.  ``p``, ``idx``, ``pos``, ``seg``, ``tiles``, ``row_tok`` and ``counts`` are the raw route's
  bits on the same logits.  ``w`` is within ``(k + 2) 2^-24 w64`` of ``w64 = p_sel / sum p_sel`` computed in fp64 from
  the kernel's own fp32 ``p`` (k - 1 fp32 additions of positive terms and one correctly rounded division).  A row with
  a NaN or Inf logit gets k distinct valid experts and NaN weights.
- Router backward with ``norm_topk``, against fp64 autograd of softmax -> gather -> renormalise from the kernel's
  ``p``: ``|got - ref| <= 2^-8 |ref| + 2 (E/32 + k + 8) 2^-24 p (M + sum p M)`` with ``M = |dpsum| + (|dw_j| +
  sum_i |w_i dw_i|) / S`` at the selected experts (``|dpsum|`` elsewhere).  Two more runs give the same bits.
- Grouped GEMM at Qwen3-30B-A3B and Qwen3-235B-A22B (E 128, k 8, T 4096): the six training GEMMs, each expert's block
  bit-identical to the plain single-CTA GEMM, within the bf16 GEMM's bound (``test_gpu_moe_reference._run_gemm``).
- ``ops.moe(norm_topk_prob=True)`` end to end with the routing held at the kernel's choice, against an fp64 autograd
  graph within the running-error bound of ``test_gpu_moe_reference``, extended by the renormalisation
  (``_norm_path_bound``); a self-test shows the bound rejects the renormalisation dropped in forward and the
  ``- sum w dw`` term dropped in backward.

The measured use of each bound is printed (``-s``).
"""
import math

import pytest
import torch
import torch.nn.functional as F

from distributed_training_guide_b200 import _ext
from test_gpu_moe_kernels import _check_layout
from test_gpu_moe_reference import (BF16, NAMES, PATH_SLACK, U, _C, _gen, _moe_inputs, _p_bound, _route, _run_gemm,
                                    _same_bits, _training_gemms)

pytestmark = pytest.mark.gpu

QWEN3_30B = dict(E=128, k=8, H=2048, I=768, T=4096)
QWEN3_235B = dict(E=128, k=8, H=4096, I=1536, T=4096)
DEBUG = dict(E=16, k=4, H=256, I=128, T=512)
NORM_MUTATIONS = ("no-renorm", "no-wdw")


# ------------------------------------------------------------------------------------------------------------------
# fp64 references (also checked without a GPU in test_qwen3_moe_cpu.py)
# ------------------------------------------------------------------------------------------------------------------
def moe_fixed_ref_norm(x, gate_w, gate_up, down, idx, logits=None, mutate=None):
    """ops.moe(norm_topk_prob=True) as an autograd graph with the experts ``idx`` [T, k] held fixed: ``y = sum_slot
    w[t, slot] expert_idx(x_t)``, ``w = p_sel / sum p_sel``, ``p = softmax(logits)``; ``logits`` as in
    ``test_gpu_moe_reference.moe_fixed_ref``.  ``mutate``: "no-renorm" weights by p_sel, "no-wdw" holds the sum
    constant (the backward loses its ``- sum w dw`` term).  Returns (y, psum)."""
    lin = x @ gate_w.t()
    lg = lin if logits is None else lin + (logits.to(lin.dtype) - lin).detach()
    p = torch.softmax(lg, -1)
    psel = p.gather(1, idx.long())
    S = psel.sum(-1, keepdim=True)
    w = psel if mutate == "no-renorm" else psel / (S.detach() if mutate == "no-wdw" else S)
    y = torch.zeros_like(x)
    for e in range(gate_w.shape[0]):
        tok, slot = (idx == e).nonzero(as_tuple=True)
        if tok.numel() == 0:
            continue
        g, u = (x[tok] @ gate_up[e].t()).chunk(2, dim=-1)
        y = y.index_add(0, tok, ((F.silu(g) * u) @ down[e].t()) * w[tok, slot, None])
    return y, p.sum(0)


def moe_fixed_grads_norm(x, gate_w, gate_up, down, idx, dy, dpsum, logits=None, mutate=None, dtype=torch.float64):
    """y, psum and the gradients (dx, d_gate, d_gate_up, d_down) of ``moe_fixed_ref_norm`` in ``dtype``."""
    leaves = [t.detach().to(dtype).requires_grad_() for t in (x, gate_w, gate_up, down)]
    y, psum = moe_fixed_ref_norm(*leaves, idx, logits=logits, mutate=mutate)
    grads = torch.autograd.grad((y, psum), leaves, (dy.to(dtype), dpsum.to(dtype)))
    return (y.detach(), psum.detach()) + tuple(grads)


def _norm_path_bound(x, gate_w, gate_up, down, idx, p, dy, dpsum, dtype):
    """``test_gpu_moe_reference._path_bound`` for renormalised weights: values and first-order error bounds, in units
    of U, of (y, dx, d_gate, d_gate_up, d_down).  Every bf16 rounding adds U times the rounded value's magnitude and
    errors propagate through the absolute value of each operation; the weights w = p_sel / S come from the kernel's
    fp32 p, and the router backward's dp = (dw - sum w dw) / S at the selected experts carries the errors of dw
    through |1 / S| and |w / S|.  Returns {name: (value, bound)}."""
    T, H = x.shape
    E, k = gate_w.shape[0], idx.shape[1]
    X, P, DY = x.to(dtype), p.to(dtype), dy.to(dtype)
    il = idx.long()
    S = P.gather(1, il).sum(-1, keepdim=True)
    Wn = P.gather(1, il) / S
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
        g, u = (xe @ Gw.t()).chunk(2, -1)
        Mg, Mu = g.abs(), u.abs()
        sg = torch.sigmoid(g)
        s0 = g * sg
        s1 = sg * (1 + g * (1 - sg))
        s2 = sg * (1 - sg) * (2 + g * (1 - 2 * sg))
        h = s0 * u
        Mh = h.abs() + (s1 * u).abs() * Mg + s0.abs() * Mu
        yp = h @ Dw.t()
        Myp = yp.abs() + Mh @ Dw.abs().t()
        we = Wn[tok, slot][:, None]
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
    wdw = (Wn * dW).sum(-1, keepdim=True)
    Mwdw = (Wn * MdW).sum(-1, keepdim=True)
    dp = dpsum.to(dtype)[None].repeat(T, 1).scatter_add_(1, il, (dW - wdw) / S)
    Mdp = z(T, E).scatter_add_(1, il, (MdW + Mwdw) / S)
    dl = P * (dp - (P * dp).sum(-1, keepdim=True))
    Mdl = dl.abs() + P * (Mdp + (P * Mdp).sum(-1, keepdim=True))
    GW = gate_w.to(dtype)
    dX = dX1 + dl @ GW
    MdX = dX.abs() + MdX1 + Mdl @ GW.abs()
    dG = dl.t() @ X
    MdG = dG.abs() + Mdl.t() @ X.abs()
    return {"y": (Y, MY), "dx": (dX, MdX), "d_gate": (dG, MdG), "d_gate_up": (dGU, MdGU), "d_down": (dDN, MdDN)}


# ------------------------------------------------------------------------------------------------------------------
# route with renormalised weights
# ------------------------------------------------------------------------------------------------------------------
TABLES = ("p", "idx", "pos", "seg", "tiles", "row_tok", "counts")


def _tables_equal(a, b, tag):
    """Every routing table of two routes bit for bit; row_tok only below seg[E], the rows the route writes."""
    for name in TABLES:
        u, v = a[name], b[name]
        if name == "row_tok":
            used = int(a["seg"][-1])
            u, v = u[:used], v[:used]
        assert _same_bits(u, v), f"{tag}: {name} differs"


def _route_norm(lg, k):
    p, idx, w, pos, seg, tiles, row_tok, counts = _C().moe_route(lg, k, True)
    torch.cuda.synchronize()
    return dict(p=p, idx=idx, w=w, pos=pos, seg=seg, tiles=tiles, row_tok=row_tok, counts=counts)


def _check_norm_route(lg, k, tag):
    """The renormalised route against the raw one (every table bit for bit) and w against fp64; returns the bound
    use."""
    raw = _route(lg, k)
    got = _route_norm(lg, k)
    _tables_equal(got, {name: getattr(raw, name) for name in TABLES}, f"{tag} (against the raw route)")
    _check_layout(got["idx"], lg.shape[1], got["pos"], got["seg"], got["tiles"], got["row_tok"], got["counts"])
    psel = raw.p.double().gather(1, raw.idx.long())
    w64 = psel / psel.sum(-1, keepdim=True)
    finite = torch.isfinite(w64).all(-1)
    assert bool(torch.isnan(got["w"][~finite]).all()), f"{tag}: a NaN row has a non-NaN weight"
    bound = (k + 2) * 2.0 ** -24 * w64[finite]
    err = (got["w"][finite].double() - w64[finite]).abs()
    assert not bool(torch.isnan(err).any()), f"{tag}: NaN weight in a finite row"
    use = (err / bound.clamp_min(1e-300)).max().item() if err.numel() else 0.0
    assert use <= 1.0, f"{tag}: w needs {use:.3g} of its bound"
    print(f"\nnorm route {tag}: w uses {use:.3g} of its bound")
    return got, raw


@pytest.mark.parametrize("T,E,k", [(T, E, k) for E, k in [(128, 8), (16, 4), (1, 1), (8, 8), (33, 33), (255, 7),
                                                          (256, 256), (256, 8)] for T in (31, 33)]
                         + [(4096, 128, 8), (131072, 128, 8), (131072, 256, 8)])
def test_norm_route_against_raw_and_fp64(T, E, k):
    lg = (torch.randn(T, E, device="cuda", generator=_gen(T + E + k)) * 3).to(BF16)
    _check_norm_route(lg, k, f"T{T} E{E} k{k}")


def test_norm_route_underflow_ties_and_non_finite_rows():
    T, E, k = 128, 128, 8
    lg = torch.randn(T, E, device="cuda", generator=_gen(3))
    lg[0:32] = -200.0 + 0.25 * torch.arange(E, device="cuda")      # one nonzero probability, the rest exact zeros
    lg[0:32, 17] = 10.0
    lg[32:64] = 0.0                                                # all tied
    lg[48:64, ::2] = 2.0
    lg[64, 5] = float("nan")
    lg[65, 9] = float("inf")
    lg[66, :] = float("-inf")
    lg[67, 3] = float("-inf")                                      # finite row: one expert at probability 0
    got, raw = _check_norm_route(lg.to(BF16), k, "underflow/ties/non-finite")
    w = got["w"]
    assert bool((w[0:32, 0] == 1.0).all()) and bool((w[0:32, 1:] == 0).all())   # 1 / 1 and 0 / 1 exactly
    assert got["idx"][0].tolist() == [17] + list(range(7))
    assert torch.equal(w[32], torch.full((k,), 0.125, device="cuda"))           # eight ties: exactly 1/8 each
    for t in (64, 65, 66):
        assert bool(torch.isnan(w[t]).all()), t
        assert len(set(got["idx"][t].tolist())) == k and all(0 <= e < E for e in got["idx"][t].tolist())
    assert bool(torch.isfinite(w[67]).all())


def test_norm_route_k_equals_e_sums_to_one():
    """k = E: every expert is selected, S is the whole row's sum, and the weights are p / S."""
    T, E = 100, 256
    lg = (torch.randn(T, E, device="cuda", generator=_gen(8)) * 2).to(BF16)
    got, _ = _check_norm_route(lg, E, "k = E = 256")
    assert bool(((got["w"].double().sum(-1) - 1).abs() < 1e-5).all())


def test_norm_route_strided_logits():
    T, E, k = 1000, 128, 8
    full = torch.randn(T, E + 40, device="cuda", generator=_gen(4)).to(BF16)
    lg = full[:, 3:3 + E]
    assert lg.stride(0) == E + 40
    a, _ = _check_norm_route(lg, k, "strided")
    b = _route_norm(lg.contiguous(), k)
    _tables_equal(a, b, "strided")
    assert _same_bits(a["w"], b["w"])


# ------------------------------------------------------------------------------------------------------------------
# router backward with renormalised weights
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("E,k", [(16, 4), (128, 8), (256, 8), (64, 64)])
@pytest.mark.parametrize("with_dpsum", [False, True])
def test_norm_router_backward_against_fp64(E, k, with_dpsum):
    C = _C()
    T = 500
    r = _route(torch.randn(T, E, device="cuda", generator=_gen(E + k)).to(BF16), k)
    dw = torch.randn(T, k, device="cuda", generator=_gen(1)) * 10
    dpsum = torch.randn(E, device="cuda", generator=_gen(2)) * 10 if with_dpsum else None
    dl = C.moe_router_bwd(r.p, r.idx, dw, dpsum, True)
    for _ in range(2):
        assert _same_bits(C.moe_router_bwd(r.p, r.idx, dw, dpsum, True), dl), "not bit-identical on a repeat"
    il = r.idx.long()
    z = torch.log(r.p.double()).requires_grad_()                   # softmax(z) is the kernel's p in fp64
    p = torch.softmax(z, -1)
    psel = p.gather(1, il)
    w = psel / psel.sum(-1, keepdim=True)
    L = (w * dw.double()).sum() + ((p * dpsum.double()).sum() if with_dpsum else 0.0)
    (ref,) = torch.autograd.grad(L, z)
    p, w, S = p.detach(), w.detach(), psel.detach().sum(-1, keepdim=True)
    M = torch.zeros(T, E, device="cuda", dtype=torch.float64) if dpsum is None else dpsum.double().abs()[None].repeat(T, 1)
    M.scatter_add_(1, il, (dw.double().abs() + (w * dw.double()).abs().sum(-1, keepdim=True)) / S)
    bound = U * ref.abs() + 2 * (E / 32 + k + 8) * 2.0 ** -24 * p * (M + (p * M).sum(-1, keepdim=True))
    use = ((dl.double() - ref).abs() / bound.clamp_min(1e-300)).max().item()
    assert use <= 1.0, use
    if k < E:   # the renormalisation matters (at k = E, S = 1 and the softmax backward cancels the - sum w dw shift)
        raw = C.moe_router_bwd(r.p, r.idx, dw, dpsum)
        assert ((raw.double() - ref).abs() > bound).any()
    print(f"\nnorm router backward E{E} k{k} dpsum={with_dpsum}: {use:.3g} of the bound")


# ------------------------------------------------------------------------------------------------------------------
# grouped GEMM at Qwen3-MoE's shapes
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("geometry", ["30B-A3B", "235B-A22B"])
@pytest.mark.parametrize("name,mode,i", [(n, m, i) for i, (n, m, _, _) in enumerate(_training_gemms(1, 1))])
def test_grouped_gemm_qwen3_moe(geometry, name, mode, i):
    d = QWEN3_30B if geometry == "30B-A3B" else QWEN3_235B
    _, _, d0, d1 = _training_gemms(d["H"], d["I"])[i]
    r = _route(torch.randn(d["T"], d["E"], device="cuda", generator=_gen(50)).to(BF16), d["k"])
    assert r.R == 49024                                            # T k + 127 E = 383 row tiles
    _run_gemm(f"Qwen3-{geometry} {name}", mode, r, d0, d1, seed=60 + mode)
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------------------------
# ops.moe(norm_topk_prob=True) end to end with the routing held fixed
# ------------------------------------------------------------------------------------------------------------------
def _kernel_moe_norm(x, gate_w, gate_up, down, k, dy, dpsum):
    from distributed_training_guide_b200 import ops

    leaves = [t.clone().requires_grad_() for t in (x, gate_w, gate_up, down)]
    n0 = _ext.launch_count()
    y, psum, counts = ops.moe(*leaves, k, norm_topk_prob=True)
    grads = torch.autograd.grad((y, psum), leaves, (dy, dpsum))
    assert _ext.launch_count() > n0, "ops.moe did not run the sm_90a kernels"
    return (y.detach(), psum.detach()) + tuple(grads)


@pytest.mark.parametrize("geometry", ["debug-qwen3-moe", "Qwen3-30B-A3B"])
def test_ops_moe_norm_fixed_routing_against_fp64(geometry):
    from distributed_training_guide_b200 import ops

    d = DEBUG if geometry == "debug-qwen3-moe" else QWEN3_30B
    E, k, H, I, T = d["E"], d["k"], d["H"], d["I"], d["T"]
    x, gate_w, gate_up, down, dy_random, dpsum = _moe_inputs(E, k, H, I, T, seed=21)
    logits = ops.gemm(x, gate_w, trans_b=True)
    r = _route(logits, k)
    # two upstream gradients: a random one, and y itself (the gradient of |y|^2 / 2), under which the routing weights'
    # gradients share a sign and the renormalisation's - sum w dw term cannot cancel
    y0 = _kernel_moe_norm(x, gate_w, gate_up, down, k, dy_random, dpsum)[0]
    for upstream, dy in (("random dy", dy_random), ("dy = y", y0)):
        got = dict(zip(NAMES, _kernel_moe_norm(x, gate_w, gate_up, down, k, dy, dpsum)))
        ref = dict(zip(NAMES, moe_fixed_grads_norm(x, gate_w, gate_up, down, r.idx, dy, dpsum, logits=logits)))
        bounds = _norm_path_bound(x, gate_w, gate_up, down, r.idx, r.p, dy, dpsum, torch.float32)
        report = []
        for name in ("y", "dx", "d_gate", "d_gate_up", "d_down"):
            b = bounds[name][1].double() * (U * PATH_SLACK)
            err = (got[name].double() - ref[name]).abs()
            use = torch.where(torch.isnan(err), torch.full_like(err, float("inf")),
                              err / b.clamp_min(1e-300)).max().item()
            report.append(f"{name} {use:.3g}")
            assert use <= 1.0, f"{geometry} {upstream} {name}: an element needs {use:.3g} of the bound"
        p64 = torch.softmax(logits.double(), -1)
        pb = _p_bound(logits, p64).sum(0) + (T / 8 + 8) * 2.0 ** -24 * p64.sum(0)
        use = ((got["psum"].double() - ref["psum"]).abs() / pb).max().item()
        report.append(f"psum {use:.3g}")
        assert use <= 1.0, f"{geometry} psum: {use:.3g} of the bound"
        print(f"\nops.moe norm_topk_prob {geometry} fixed routing, {upstream}, bound use: " + ", ".join(report))
    if geometry != "debug-qwen3-moe":
        return
    for m in NORM_MUTATIONS:   # with dy = y
        bad = dict(zip(NAMES, moe_fixed_grads_norm(x, gate_w, gate_up, down, r.idx, dy, dpsum, logits=logits,
                                                   mutate=m)))
        caught = [n for n in ("y", "dx", "d_gate", "d_gate_up", "d_down")
                  if ((got[n].double() - bad[n]).abs() > bounds[n][1].double() * (U * PATH_SLACK)).any()]
        print(f"mutation {m}: rejected by {caught}")
        assert caught, f"the bound does not reject {m}"


def test_ops_moe_norm_is_bit_identical_run_to_run():
    d = DEBUG
    x, gate_w, gate_up, down, dy, dpsum = _moe_inputs(d["E"], d["k"], d["H"], d["I"], d["T"], seed=22)
    a = _kernel_moe_norm(x, gate_w, gate_up, down, d["k"], dy, dpsum)
    b = _kernel_moe_norm(x, gate_w, gate_up, down, d["k"], dy, dpsum)
    for n, u, v in zip(NAMES, a, b):
        assert _same_bits(u, v), n


def test_ops_moe_flag_off_is_the_raw_path():
    """norm_topk_prob=False launches what ops.moe launched before the flag existed: the same bits as the default."""
    from distributed_training_guide_b200 import ops

    d = DEBUG
    x, gate_w, gate_up, down, dy, dpsum = _moe_inputs(d["E"], d["k"], d["H"], d["I"], d["T"], seed=23)
    outs = []
    for kw in ({}, {"norm_topk_prob": False}):
        leaves = [t.clone().requires_grad_() for t in (x, gate_w, gate_up, down)]
        n0 = _ext.launch_count()
        y, psum, _ = ops.moe(*leaves, d["k"], **kw)
        grads = torch.autograd.grad((y, psum), leaves, (dy, dpsum))
        outs.append(((y, psum) + grads, _ext.launch_count() - n0))
    assert outs[0][1] == outs[1][1]
    for n, u, v in zip(NAMES, outs[0][0], outs[1][0]):
        assert _same_bits(u, v), n
