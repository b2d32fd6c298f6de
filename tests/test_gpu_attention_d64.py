"""The head_dim-64 wgmma attention kernels (``attn_fwd(..., head_dim=64)`` versions 1 and 2, ``attn_bwd(...,
head_dim=64)`` modes 1 and 2, each plain causal, with document masking, with a sliding window and with both) against
fp64, element by element, with the bounds of ``test_gpu_attention_reference.py``: ``2^-8`` for the bf16 roundings,
``n 2^-24`` for fp32 accumulation over n keys (queries) and the fp32 error of the 64-long dot products, no outlier
budget; and the worst 128-row tile against the correctly rounded flash attention (and PyTorch's FA2 where it applies).

The fp64 references here take the head dim from the tensors; only helpers that do not depend on it are imported.
Exact structural checks follow: inputs a row cannot see leave its outputs bit-identical, a NaN reaches exactly the
outputs that depend on it, repeated calls are bit-identical, and every head_dim / shape mismatch is refused before any
launch.  ``ops.attention_qkv`` at d = 64 runs the kernels through autograd, and keeps the SDPA fallback at S 200."""
import math

import pytest
import torch

from distributed_training_guide_b200 import _ext, ops
from test_gpu_attention_reference import (C_DK, C_DQ, C_DV, C_LSE, C_O, DOC_CUTS, U, _bits_equal, _block_any,
                                          _check_tiles, _chunks, _docs, _elem_c, _flash_sdpa, _heads, _lse_c,
                                          _misaligned, _refused, _visible)

pytestmark = pytest.mark.gpu
DEV = "cuda"
BF16 = torch.bfloat16
D = 64
SC = 1.0 / math.sqrt(D)


def _C():
    return _ext.load(True)


def _inputs(B, S, nh, nkv, pattern, scale, seed=0, d=D):
    """qkv [B, S, nh + 2 nkv, d] and dO [B, S, nh, d] in bf16, with values of the named pattern."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(B, S, nh + 2 * nkv, d, device=DEV, generator=g)
    do = torch.randn(B, S, nh, d, device=DEV, generator=g)
    q, k, v = x[:, :, :nh], x[:, :, nh:nh + nkv], x[:, :, nh + nkv:]
    if pattern == "peaked":       # scaled scores with a standard deviation of 30: most p underflow
        sd = math.sqrt(30.0 / (scale * math.sqrt(d)))
        q.mul_(sd)
        k.mul_(sd)
    elif pattern == "sink":       # key 0 beats every other key of every query by >= 8 scaled score units
        u = torch.randint(0, 2, (d,), device=DEV, generator=g).float() * 2 - 1
        q.add_(u)
        k[:, 0] = u * ((8.0 + 64.0 * scale) / (d * scale))
    elif pattern == "late_max":   # row maxima that jump in late key blocks, for some rows of a warp only
        boost = torch.ones(S, device=DEV)
        boost[3 * S // 10:3 * S // 10 + 10] = 5.0
        boost[7 * S // 10:] = 9.0
        rows = torch.ones(S, device=DEV)
        rows[::3] = 0.05
        k.mul_(boost[None, :, None, None])
        q.mul_(rows[None, :, None, None])
    elif pattern == "offset_v":   # a large common offset: l (fp32, unrounded p) must match the bf16 P that meets V
        v.add_(64.0)
    else:
        assert pattern == "normal", pattern
    return x.to(BF16), do.to(BF16)


# ------------------------------------------------------------------------------------------------------------------
# fp64 references (the head dim is qkv's last dimension)
# ------------------------------------------------------------------------------------------------------------------
def _fwd64(qkv, nh, nkv, scale, ds=None, window=None):
    """Exact O and lse, the companion P |V|, the score term, the visible-key count n and the correctly rounded flash
    attention's O (P rounded to bf16 with the final row max).  Tensors are [B, nh, S, d] / [B, nh, S]."""
    B, S, _, d = qkv.shape
    q, k, v = _heads(qkv, nh, nkv)
    r = {name: torch.empty(B, nh, S, d, device=DEV, dtype=torch.float64) for name in ("o", "comp", "score", "yard")}
    r["lse"] = torch.empty(B, nh, S, device=DEV, dtype=torch.float64)
    r["n"] = torch.empty(B, 1, S, 1, device=DEV, dtype=torch.float64)
    c0 = d * U * scale
    for r0, r1, k0 in _chunks(B, S, nh, ds, window):
        kk, vv = k[:, :, k0:r1], v[:, :, k0:r1]
        vis = _visible(ds, r0, r1, k0, r1, window)[:, None]
        qr = q[:, :, r0:r1]
        s = (qr @ kk.transpose(-1, -2)).mul_(scale).masked_fill_(~vis, float("-inf"))
        m = s.amax(-1, keepdim=True)
        e = s.sub_(m).exp_()
        l = e.sum(-1, keepdim=True)
        r["lse"][:, :, r0:r1] = (m + l.log()).squeeze(-1)
        r["yard"][:, :, r0:r1] = (e.to(BF16).double() @ vv) / l
        p = e.div_(l)
        o = p @ vv
        r["o"][:, :, r0:r1] = o
        r["comp"][:, :, r0:r1] = p @ vv.abs()
        a = p.mul_(qr.abs() @ kk.abs().transpose(-1, -2))   # P o (|Q||K|^T)
        r["score"][:, :, r0:r1] = (a @ vv.abs() + a.sum(-1, keepdim=True) * o.abs()) * c0
        r["n"][:, 0, r0:r1, 0] = vis.sum(-1).double().expand(B, 1, -1)[:, 0]
        del s, e, p, a, o
    r["yard"] = r["yard"].to(BF16)
    return r


def _bwd64(qkv, do, o, lse, nh, nkv, scale, ds=None, window=None):
    """Exact dQ / dK / dV of the flash-backward formula on the given ``o`` [B, S, nh, d] and ``lse`` [B, nh, S],
    their companions, score terms, accumulation counts and the correctly rounded flash backward's gradients."""
    B, S, _, d = qkv.shape
    g = nh // nkv
    q, k, v = _heads(qkv, nh, nkv)
    dO = do.double().permute(0, 2, 1, 3)
    o64 = o.double().permute(0, 2, 1, 3)
    delta = (dO * o64).sum(-1, keepdim=True)
    dabs = (dO.abs() * o64.abs()).sum(-1, keepdim=True)
    lse = lse.double()[..., None]
    z = lambda: torch.zeros(B, nh, S, d, device=DEV, dtype=torch.float64)  # noqa: E731
    r = {name: z() for name in ("dq", "dq_comp", "dq_score", "dq_yard", "dk", "dk_comp", "dk_score", "dk_yard",
                                "dv", "dv_comp", "dv_score", "dv_yard")}
    nq = torch.zeros(B, 1, S, 1, device=DEV, dtype=torch.float64)
    nk = torch.zeros(B, 1, S, 1, device=DEV, dtype=torch.float64)
    c0 = d * U * scale
    for r0, r1, k0 in _chunks(B, S, nh, ds, window):
        kk, vv = k[:, :, k0:r1], v[:, :, k0:r1]
        vis = _visible(ds, r0, r1, k0, r1, window)[:, None]
        qr, dOr = q[:, :, r0:r1], dO[:, :, r0:r1]
        s = (qr @ kk.transpose(-1, -2)).mul_(scale)
        p = s.sub_(lse[:, :, r0:r1]).exp_().masked_fill_(~vis, 0.0)
        t = (dOr @ vv.transpose(-1, -2)).sub_(delta[:, :, r0:r1])
        ds_ = p * t * scale
        pt, dst = p.transpose(-1, -2), ds_.transpose(-1, -2)
        r["dv"][:, :, k0:r1] += pt @ dOr
        r["dv_comp"][:, :, k0:r1] += pt @ dOr.abs()
        r["dk"][:, :, k0:r1] += dst @ qr
        r["dk_comp"][:, :, k0:r1] += dst.abs() @ qr.abs()
        r["dq"][:, :, r0:r1] = ds_ @ kk
        r["dq_comp"][:, :, r0:r1] = ds_.abs() @ kk.abs()
        r["dv_yard"][:, :, k0:r1] += p.to(BF16).double().transpose(-1, -2) @ dOr
        dsb = ds_.to(BF16).double()
        r["dk_yard"][:, :, k0:r1] += dsb.transpose(-1, -2) @ qr
        r["dq_yard"][:, :, r0:r1] = dsb @ kk
        del dsb, ds_, dst
        a = qr.abs() @ kk.abs().transpose(-1, -2)
        ep = (p * a).mul_(c0)                                         # error base of P
        es = a.mul_(t.abs_()).mul_(scale).add_(dOr.abs() @ vv.abs().transpose(-1, -2)).add_(dabs[:, :, r0:r1])
        es.mul_(p).mul_(c0)                                           # error base of dS
        r["dv_score"][:, :, k0:r1] += ep.transpose(-1, -2) @ dOr.abs()
        r["dk_score"][:, :, k0:r1] += es.transpose(-1, -2) @ qr.abs()
        r["dq_score"][:, :, r0:r1] = es @ kk.abs()
        nq[:, 0, r0:r1, 0] = vis.sum(-1).double().expand(B, 1, -1)[:, 0]
        nk[:, 0, k0:r1, 0] += vis.sum(-2).double().expand(B, 1, -1)[:, 0]
        del s, p, t, a, ep, es
    out = {}
    for name, val in r.items():
        out[name] = val if name.startswith("dq") else val.view(B, nkv, g, S, d).sum(2)
    for name in ("dq_yard", "dk_yard", "dv_yard"):
        out[name] = out[name].to(BF16)
    out["nq"], out["nk"] = nq, nk * g
    return out


# ------------------------------------------------------------------------------------------------------------------
# the kernels against fp64
# ------------------------------------------------------------------------------------------------------------------
# (B, S, nh, nkv, scale, pattern, documents, window)
CASES = {
    "one-tile": (1, 128, 1, 1, SC, "normal", None, None),
    "b3-4:4-scale-0.05": (3, 384, 4, 4, 0.05, "normal", None, None),
    "16:1-sink": (2, 384, 16, 1, SC, "sink", None, None),
    "llama-3.2-1b-4096": (1, 4096, 32, 8, SC, "normal", None, None),
    "9:3-late-max": (1, 4096, 9, 3, SC, "late_max", None, None),
    "32:8-peaked-scale-1": (1, 384, 32, 8, 1.0, "peaked", None, None),
    "docs-offset-v": (2, 4096, 4, 2, SC, "offset_v", "edges", None),
    "docs-9:3-peaked": (2, 384, 9, 3, SC, "peaked", "edges", None),
    "one-token-docs": (2, 384, 4, 4, SC, "normal", "tokens", None),
    "w1": (2, 384, 4, 2, SC, "normal", None, 1),
    "w127-peaked": (1, 4096, 4, 1, SC, "peaked", None, 127),
    "w129-offset-v": (1, 384, 8, 2, 1.0, "offset_v", None, 129),
    "wS-1-sink": (1, 384, 16, 1, SC, "sink", None, 383),
    "w4095-32:8": (1, 4096, 32, 8, SC, "normal", None, 4095),
    "docs-w129": (2, 4096, 9, 3, SC, "normal", "edges", 129),
    "docs-w127-late-max": (2, 384, 16, 1, 0.05, "late_max", "edges", 127),
    "docs-w1-4:4": (2, 128, 4, 4, SC, "normal", "edges", 1),
}


@pytest.mark.parametrize("case", list(CASES))
def test_d64_kernels_against_fp64(case):
    B, S, nh, nkv, scale, pattern, layout, window = CASES[case]
    C = _C()
    qkv, do = _inputs(B, S, nh, nkv, pattern, scale, seed=len(case))
    ds = _docs(B, S, layout)
    plain = ds is None and window is None
    f = _fwd64(qkv, nh, nkv, scale, ds, window)
    sdpa = _flash_sdpa(qkv, do, nh, nkv, scale) if plain else None
    lines = []
    for version in (1, 2):
        o, lse = C.attn_fwd(qkv, nh, nkv, scale, version, doc_start=ds, window=window, head_dim=D)
        assert o.shape == (B, S, nh, D)
        ot = o.permute(0, 2, 1, 3)
        c = _elem_c(ot, f["o"], f["comp"], f["score"], f["n"])
        cl = _lse_c(lse, f["lse"])
        yards = {"rounded": f["yard"], **({"FA2": sdpa[0]} if plain else {})}
        lines.append(f"fwd v{version}: O c {c:.3g}  lse c {cl:.3g}  {_check_tiles(f'{case} v{version} O', ot, f['o'], yards)}")
        assert c <= C_O, f"{case} v{version}: an element of O needs c = {c:.3g} > {C_O}"
        assert cl <= C_LSE, f"{case} v{version}: an lse element needs c = {cl:.3g} > {C_LSE}"
    del o, lse, ot
    o_in = f["o"].to(BF16).permute(0, 2, 1, 3).contiguous()
    lse_in = f["lse"].float()
    del f
    b = _bwd64(qkv, do, o_in, lse_in, nh, nkv, scale, ds, window)
    sl = {"dq": slice(0, nh), "dk": slice(nh, nh + nkv), "dv": slice(nh + nkv, nh + 2 * nkv)}
    cmax = {"dq": C_DQ, "dk": C_DK, "dv": C_DV}
    for mode in (1, 2):
        g = C.attn_bwd(do, qkv, o_in, lse_in, nh, nkv, scale, None, mode, doc_start=ds, window=window, head_dim=D)
        assert g.shape == qkv.shape
        for i, name in enumerate(("dq", "dk", "dv")):
            got = g[:, :, sl[name]].permute(0, 2, 1, 3)
            n = b["nq"] if name == "dq" else b["nk"]
            c = _elem_c(got, b[name], b[name + "_comp"], b[name + "_score"], n)
            yards = {"rounded": b[name + "_yard"], **({"FA2": sdpa[1 + i]} if plain else {})}
            lines.append(f"bwd mode {mode} {name}: c {c:.3g}  "
                         f"{_check_tiles(f'{case} mode {mode} {name}', got, b[name], yards)}")
            assert c <= cmax[name], f"{case} mode {mode}: an element of {name} needs c = {c:.3g} > {cmax[name]}"
    print(f"\n{case}:\n  " + "\n  ".join(lines))


# ------------------------------------------------------------------------------------------------------------------
# exact structural checks
# ------------------------------------------------------------------------------------------------------------------
SB, SS, SNH, SNKV, SW = 2, 512, 4, 2, 129
MASKS = {"plain": (None, None), "docs": ("edges", None), "window": (None, SW), "docs+window": ("edges", SW)}


def _struct_mask(mask):
    layout, window = MASKS[mask]
    return _docs(SB, SS, layout), window


def _vis_all(ds, window):
    return _visible(ds, 0, SS, 0, SS, window).expand(SB, SS, SS)


def _run(qkv, do, ds, window, version, mode):
    C = _C()
    o, lse = C.attn_fwd(qkv, SNH, SNKV, SC, version, doc_start=ds, window=window, head_dim=D)
    g = C.attn_bwd(do, qkv, o, lse, SNH, SNKV, SC, None, mode, doc_start=ds, window=window, head_dim=D)
    return o, lse, g


@pytest.mark.parametrize("mask", list(MASKS))
def test_d64_invisible_keys_and_queries_do_not_matter(mask):
    """Replacing K and V of key p leaves O, lse and dQ of every row that cannot see p unchanged, bit for bit;
    replacing Q and dO of query p leaves dK and dV of every key p cannot see unchanged."""
    ds, window = _struct_mask(mask)
    vis = _vis_all(ds, window)                          # [B, q, k]
    qkv, do = _inputs(SB, SS, SNH, SNKV, "normal", SC, seed=21)
    extra = set()
    if ds is not None:
        extra |= {c - 1 for c in DOC_CUTS[0] if 0 < c < SS}
    if window is not None:
        extra |= {SS - 1 - window, SS - window, 200 - window}
    positions = sorted({1, 63, 64, 127, 128, 129, 191, SS - 1} | {p for p in extra if 0 <= p < SS})
    gen = torch.Generator(device=DEV).manual_seed(22)
    for version, mode in ((1, 1), (2, 2)):
        o0, l0, g0 = _run(qkv, do, ds, window, version, mode)
        for p in positions:
            x = qkv.clone()
            x[:, p, SNH:] = torch.randn(SB, 2 * SNKV, D, device=DEV, generator=gen).to(BF16)
            o1, l1, g1 = _run(x, do, ds, window, version, mode)
            blind = ~vis[:, :, p]                        # [B, q]: rows that cannot see key p
            assert _bits_equal(o1[blind], o0[blind]), (mask, version, "O", p)
            assert _bits_equal(l1.permute(0, 2, 1)[blind], l0.permute(0, 2, 1)[blind]), (mask, version, "lse", p)
            assert _bits_equal(g1[:, :, :SNH][blind], g0[:, :, :SNH][blind]), (mask, mode, "dQ", p)
            assert not torch.equal(o1[:, p], o0[:, p]), (mask, version, "row p sees key p", p)
            x = qkv.clone()
            d1 = do.clone()
            x[:, p, :SNH] = torch.randn(SB, SNH, D, device=DEV, generator=gen).to(BF16)
            d1[:, p] = torch.randn(SB, SNH, D, device=DEV, generator=gen).to(BF16)
            o1, l1, g1 = _run(x, d1, ds, window, version, mode)
            blind = ~vis[:, p, :]                        # [B, k]: keys query p cannot see
            assert _bits_equal(g1[:, :, SNH:][blind], g0[:, :, SNH:][blind]), (mask, mode, "dK/dV", p)


@pytest.mark.parametrize("mask", list(MASKS))
def test_d64_nan_reaches_exactly_the_outputs_that_depend_on_it(mask):
    """A NaN in K of key k makes O and lse NaN exactly at the rows of the group that see k; a NaN in V of key k makes
    dK NaN at exactly that key; a NaN in dO of query q makes dQ NaN at exactly that query.  The gradient MMAs also
    multiply the masked entries of a processed block, so the NaN may reach dQ (dK / dV) only inside blocks the kernel
    processes: it must stay outside every 128 x 64 block with no visible pair, which shows the block skipping."""
    ds, window = _struct_mask(mask)
    vis = _vis_all(ds, window)
    g = SNH // SNKV
    qkv, do = _inputs(SB, SS, SNH, SNKV, "normal", SC, seed=31)
    for version, mode in ((1, 2), (2, 1)):
        for b, h, k in ((0, 0, 0), (1, 1, 129), (0, 1, 300), (1, 0, SS - 1)):
            heads = torch.zeros(SNH, dtype=torch.bool, device=DEV)
            heads[h * g:(h + 1) * g] = True
            want = torch.zeros(SB, SS, SNH, dtype=torch.bool, device=DEV)
            want[b] = vis[b, :, k][:, None] & heads[None, :]
            x = qkv.clone()
            x[b, k, SNH + h, 17] = float("nan")
            o, lse = _C().attn_fwd(x, SNH, SNKV, SC, version, doc_start=ds, window=window, head_dim=D)
            assert torch.equal(torch.isnan(o).any(-1), want), (mask, version, b, h, k)
            assert torch.equal(torch.isnan(o).all(-1), want), (mask, version, b, h, k)
            assert torch.equal(torch.isnan(lse), want.permute(0, 2, 1)), (mask, version, b, h, k)
            # backward, NaN in V
            o, lse = _C().attn_fwd(qkv, SNH, SNKV, SC, version, doc_start=ds, window=window, head_dim=D)
            x = qkv.clone()
            x[b, k, SNH + SNKV + h, 5] = float("nan")
            gr = _C().attn_bwd(do, x, o, lse, SNH, SNKV, SC, None, mode, doc_start=ds, window=window, head_dim=D)
            bad = torch.isnan(gr).any(-1)
            want_k = torch.zeros(SB, SS, SNKV, dtype=torch.bool, device=DEV)
            want_k[b, k, h] = True
            assert torch.equal(bad[:, :, SNH:SNH + SNKV], want_k), (mask, mode, "dK", b, h, k)
            assert not bad[:, :, SNH + SNKV:].any(), (mask, mode, "dV", b, h, k)
            dq_bad = bad[:, :, :SNH]
            assert not dq_bad[:, :, ~heads].any() and not dq_bad[1 - b].any(), (mask, mode, b, h, k)
            assert dq_bad[b][vis[b, :, k]][:, heads].all(), (mask, mode, "dQ where real", b, h, k)
            seen = _block_any(vis[b:b + 1], 128, 64)[0, :, k // 64]            # [S/128]: blocks processed with k
            assert not dq_bad[b].view(SS // 128, 128, SNH)[~seen].any(), (mask, mode, "dQ outside", b, h, k)
            # backward, NaN in dO of query k (head hq)
            hq = h * g + 1
            d1 = do.clone()
            d1[b, k, hq, 9] = float("nan")
            gr = _C().attn_bwd(d1, qkv, o, lse, SNH, SNKV, SC, None, mode, doc_start=ds, window=window, head_dim=D)
            bad = torch.isnan(gr).any(-1)
            want_q = torch.zeros(SB, SS, SNH, dtype=torch.bool, device=DEV)
            want_q[b, k, hq] = True
            assert torch.equal(bad[:, :, :SNH], want_q), (mask, mode, "dQ", b, hq, k)
            kv_bad = bad[:, :, SNH:].view(SB, SS, 2, SNKV)
            other = [i for i in range(SNKV) if i != h]
            assert not kv_bad[:, :, :, other].any() and not kv_bad[1 - b].any(), (mask, mode, b, hq, k)
            assert kv_bad[b, :, :, h][vis[b, k, :]].all(), (mask, mode, "dK/dV where real", b, hq, k)
            seen = _block_any(vis[b:b + 1].transpose(1, 2).contiguous(), 128, 64)[0, :, k // 64]
            assert not kv_bad[b, :, :, h].view(SS // 128, 128, 2)[~seen].any(), (mask, mode, "dK/dV outside", b, k)


@pytest.mark.parametrize("mask", list(MASKS))
def test_d64_repeated_calls_are_bit_identical(mask):
    ds, window = _struct_mask(mask)
    qkv, do = _inputs(SB, SS, SNH, SNKV, "normal", SC, seed=61)
    for version, mode in ((1, 1), (1, 2), (2, 1), (2, 2)):
        a = _run(qkv, do, ds, window, version, mode)
        b = _run(qkv, do, ds, window, version, mode)
        assert all(_bits_equal(x, y) for x, y in zip(a, b)), (mask, version, mode)


# ------------------------------------------------------------------------------------------------------------------
# refused arguments
# ------------------------------------------------------------------------------------------------------------------
def test_d64_binding_refuses_bad_head_dims_and_mismatched_tensors():
    C = _C()
    nh, nkv, S = 2, 1, 256
    q64, do64 = _inputs(1, S, nh, nkv, "normal", SC, seed=71)
    q128, do128 = _inputs(1, S, nh, nkv, "normal", SC, seed=72, d=128)
    o64, lse64 = C.attn_fwd(q64, nh, nkv, SC, head_dim=64)
    o128, lse128 = C.attn_fwd(q128, nh, nkv, SC)
    # head_dim outside {64, 128}, with a qkv that has that last dimension
    for hd in (0, -64, 32, 96, 256):
        x = torch.zeros(1, S, nh + 2 * nkv, max(hd, 16), device=DEV, dtype=BF16)
        for version in (1, 2):
            _refused(lambda: C.attn_fwd(x, nh, nkv, SC, version, head_dim=hd), "head_dim must be 64 or 128")
        for mode in (1, 2):
            _refused(lambda: C.attn_bwd(do64, x, o64, lse64, nh, nkv, SC, None, mode, head_dim=hd),
                     "head_dim must be 64 or 128")
    # qkv of the other width
    for version in (1, 2):
        _refused(lambda: C.attn_fwd(q128, nh, nkv, SC, version, head_dim=64), r"qkv must be \[B, S, nh\+2\*nkv, 64\]")
        _refused(lambda: C.attn_fwd(q64, nh, nkv, SC, version, head_dim=128), r"qkv must be \[B, S, nh\+2\*nkv, 128\]")
        _refused(lambda: C.attn_fwd(q64, nh, nkv, SC, version), r"qkv must be \[B, S, nh\+2\*nkv, 128\]")
    for mode in (1, 2):
        _refused(lambda: C.attn_bwd(do64, q128, o64, lse64, nh, nkv, SC, None, mode, head_dim=64),
                 r"qkv must be \[B, S, nh\+2\*nkv, 64\]")
        _refused(lambda: C.attn_bwd(do128, q64, o128, lse128, nh, nkv, SC, None, mode), r"qkv must be \[B, S")
        # o or d_o of the other width
        _refused(lambda: C.attn_bwd(do64, q64, o128, lse64, nh, nkv, SC, None, mode, head_dim=64),
                 r"(?<!\w)o must be \[B, S, nh, 64\]")
        _refused(lambda: C.attn_bwd(do128, q64, o64, lse64, nh, nkv, SC, None, mode, head_dim=64),
                 r"d_o must be \[B, S, nh, 64\]")
        _refused(lambda: C.attn_bwd(do128, q128, o64, lse128, nh, nkv, SC, None, mode, head_dim=128),
                 r"(?<!\w)o must be \[B, S, nh, 128\]")
        _refused(lambda: C.attn_bwd(do64, q128, o128, lse128, nh, nkv, SC, None, mode),
                 r"d_o must be \[B, S, nh, 128\]")
        # a 64-wide o reshaped to 128 columns
        _refused(lambda: C.attn_bwd(do64, q64, o64.reshape(1, S, nh // 2, 128).contiguous(), lse64, nh, nkv, SC,
                                    None, mode, head_dim=64), r"(?<!\w)o must be \[B, S, nh, 64\]")
    # misaligned qkv / d_o at head_dim 64
    for elems in (1, 4):
        bad = _misaligned(q64, elems)
        _refused(lambda: C.attn_fwd(bad, nh, nkv, SC, head_dim=64), "qkv must start on a 16-byte boundary")
        _refused(lambda: C.attn_bwd(do64, bad, o64, lse64, nh, nkv, SC, head_dim=64),
                 "qkv must start on a 16-byte boundary")
        bad = _misaligned(do64, elems)
        _refused(lambda: C.attn_bwd(bad, q64, o64, lse64, nh, nkv, SC, head_dim=64), "16-byte boundary")


# ------------------------------------------------------------------------------------------------------------------
# the op through autograd
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mask", ["plain", "docs+window"])
def test_attention_qkv_d64_runs_the_kernels_through_autograd(mask):
    """At Llama-3.2-1B head geometry (32:8, d 64, heads reduced to 8:2): one forward and three backward launches
    (delta, KV pass, Q pass), judged with the tile yardstick.  Plain causal: against the true fp64 gradient.  With
    short documents (and a window) the bf16 rounding of the kernels' own O inside delta = rowsum(dO o) dominates dQ
    of rows that see few keys (1.38x the yardstick on the true gradient), so the gradients are judged on the
    backward formula with that o, as the element-wise test judges the backward on its own inputs."""
    S, nh, nkv = 4096, 8, 2
    layout, window = {"plain": (None, None), "docs+window": ("edges", 1000)}[mask]
    ds = _docs(1, S, layout)
    qkv, do = _inputs(1, S, nh, nkv, "normal", SC, seed=9)
    x = qkv.clone().requires_grad_(True)
    y = x * 1.0
    torch.cuda.synchronize()
    n0 = _ext.launch_count()
    out = ops.attention_qkv(y, nh, nkv, doc_start=ds, window=window)
    torch.cuda.synchronize()
    assert _ext.launch_count() - n0 == 1
    assert out.shape == (1, S, nh, D)
    out.backward(do)
    torch.cuda.synchronize()
    assert _ext.launch_count() - n0 == 4
    f = _fwd64(qkv, nh, nkv, SC, ds, window)
    msg = [_check_tiles(f"{mask} O", out.permute(0, 2, 1, 3), f["o"], {"rounded": f["yard"]})]
    o_ref = f["o"].permute(0, 2, 1, 3) if mask == "plain" else out.detach()
    b = _bwd64(qkv, do, o_ref, f["lse"], nh, nkv, SC, ds, window)
    for name, sl in (("dq", slice(0, nh)), ("dk", slice(nh, nh + nkv)), ("dv", slice(nh + nkv, None))):
        got = x.grad[:, :, sl].permute(0, 2, 1, 3)
        msg.append(f"{name} " + _check_tiles(f"{mask} {name}", got, b[name], {"rounded": b[name + "_yard"]}))
    print(f"\n{mask}: " + "; ".join(msg))


def test_attention_qkv_d64_ragged_sequence_keeps_the_sdpa_fallback():
    S, nh, nkv = 200, 4, 2
    qkv, do = _inputs(1, S, nh, nkv, "normal", SC, seed=10)
    x = qkv.clone().requires_grad_(True)
    torch.cuda.synchronize()
    n0 = _ext.launch_count()
    out = ops.attention_qkv(x, nh, nkv)
    out.backward(do)
    torch.cuda.synchronize()
    assert _ext.launch_count() == n0
    f = _fwd64(qkv, nh, nkv, SC)
    err = ((out.permute(0, 2, 1, 3).double() - f["o"]).norm() / f["o"].norm()).item()
    assert err < 1e-2, err
