"""The wgmma attention kernels (``attn_fwd`` versions 1 and 2, ``attn_bwd`` modes 1 and 2, each plain causal, with
document masking, with a sliding window and with both) against fp64, element by element.

The fp64 reference runs on the GPU a chunk of query rows at a time, so no [S, S, heads] tensor is ever built.  The
backward is judged on its own: the kernel gets ``o = bf16(O64)`` and ``lse = fp32(lse64)``, and the reference is the
exact flash-backward formula on those same inputs (``P = exp(s*scale - lse)``, ``dS = P (dO V^T - rowsum(dO o))
scale``, ``dV = P^T dO``, ``dK = dS^T Q``, ``dQ = dS K``, the GQA group summed in fp64).

Two bounds per output, neither with an outlier budget:
- every element: ``|got - exact| <= 2^-8 |exact| + (2^-8 + c n 2^-24) companion + c score``.  ``2^-8 |exact|`` is the
  bf16 rounding of the output, ``2^-8 companion`` covers P (dS) rounded to bf16 before the second MMA, ``n 2^-24``
  the fp32 accumulation over the n visible keys (queries), and ``score`` the fp32 error of the 128-long dot products
  (``128 2^-24 scale |Q||K|^T`` propagated through P, plus ``dO V^T`` and ``rowsum(dO o)`` for dK / dQ).  The
  companions are ``P |V|`` (O), ``P^T |dO|`` (dV), ``|dS|^T |Q|`` (dK) and ``|dS| |K|`` (dQ).  lse gets
  ``|got - exact| <= c 2^-23 (1 + |exact|)``.  This is the bound that sees a single wrong element.
- worst (batch, head, 128-row tile): the relative L2 error may be at most ``TILE_FACTOR`` times that of (a) the same
  fp64 computation with P (and dS) rounded to bf16 with the final row max, a correctly rounded flash attention, and,
  for plain causal attention, (b) PyTorch's bf16 flash attention (``SDPBackend.FLASH_ATTENTION``) on the same inputs,
  plus ``TILE_SLACK``.

Exact structural checks: inputs a row cannot see do not change its outputs, bit for bit; a NaN reaches exactly the
outputs that depend on it; reads stay inside ``qkv`` and ``d_o``; W = 1 and one-token documents; and every argument
of ``attn_fwd`` / ``attn_bwd`` is checked before the first launch.
"""
import math

import pytest
import torch
from torch.nn.attention import SDPBackend, sdpa_kernel

from distributed_training_guide_b200 import _ext, ops
from distributed_training_guide_b200.ops import reference as ref
from test_gpu_attention_docmask import _doc_start

pytestmark = pytest.mark.gpu
DEV = "cuda"
BF16 = torch.bfloat16
D = 128
SC = 1.0 / math.sqrt(D)
U = 2.0 ** -24

# Measured on an H100 80GB HBM3 at a 400 W power limit over every case of this file (both forward versions and both
# backward modes give the same numbers):
# - every element: O and dV need c = 0 everywhere (the two 2^-8 terms cover every element), so their constant only
#   leaves room for the fp32 terms; dQ needs at most 9.9e-3 (70B heads, peaked rows at scale 1; 9.4e-3 at W 1), dK
#   9.3e-3 (W 1), lse 22.6 (70B heads, peaked rows at scale 1; at most 4.4 elsewhere).
# - worst tile: against the correctly rounded flash attention 0.98x to 1.005x for every output, mask and shape;
#   through autograd against the true fp64 gradient (where the kernels' own bf16 o also enters delta) up to 1.10x
#   (dQ, Mistral geometry).  Against PyTorch's FA2 (plain causal only): O 0.999x to 1.008x, gradients 0.50x to 1.000x,
#   and 0.022x for dQ with an attention sink and a GQA group of 16, where FA2's dQ is off by 15 %.
C_O, C_DV = 1e-3, 1e-3
C_DQ, C_DK = 4e-2, 4e-2
C_LSE = 100.0
TILE_FACTOR, TILE_SLACK = 1.2, 1e-5
CHUNK_ELEMS = 2 ** 24   # (batch x heads x query rows x keys) per fp64 reference chunk


def _C():
    return _ext.load(True)


# ------------------------------------------------------------------------------------------------------------------
# inputs
# ------------------------------------------------------------------------------------------------------------------
def _inputs(B, S, nh, nkv, pattern, scale, seed=0):
    """qkv [B, S, nh + 2 nkv, 128] and dO [B, S, nh, 128] in bf16, with values of the named pattern."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(B, S, nh + 2 * nkv, D, device=DEV, generator=g)
    do = torch.randn(B, S, nh, D, device=DEV, generator=g)
    q, k, v = x[:, :, :nh], x[:, :, nh:nh + nkv], x[:, :, nh + nkv:]
    if pattern == "peaked":       # scaled scores with a standard deviation of 30: most p underflow
        sd = math.sqrt(30.0 / (scale * math.sqrt(D)))
        q.mul_(sd)
        k.mul_(sd)
    elif pattern == "sink":       # key 0 beats every other key of every query by >= 8 scaled score units
        u = torch.randint(0, 2, (D,), device=DEV, generator=g).float() * 2 - 1
        q.add_(u)
        k[:, 0] = u * ((8.0 + 64.0 * scale) / (D * scale))
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
    elif pattern == "uniform":    # near-uniform rows
        q.mul_(1e-3)
        k.mul_(1e-3)
    else:
        assert pattern == "normal", pattern
    return x.to(BF16), do.to(BF16)


# documents of one token, and documents that cross 64- and 128-row edges; a different layout per batch row
DOC_CUTS = [[0, 1, 2, 3, 63, 64, 65, 127, 128, 129, 130, 191, 192, 300, 383, 384, 385, 700, 1000, 1001, 1500, 2047],
            [0, 64, 128, 250, 251, 252, 640, 641, 1023, 1100, 1600]]


def _docs(B, S, layout):
    if layout is None:
        return None
    if layout == "tokens":
        rows = [list(range(S))] * B
    else:
        rows = [[c for c in DOC_CUTS[b % 2] if c < S] for b in range(B)]
    return torch.stack([_doc_start(S, r) for r in rows]).to(DEV)


def _visible(ds, r0, r1, k0, k1, window):
    """bool [B | 1, r1 - r0, k1 - k0]: query q sees key k, ``ref.document_mask``'s rule for a block of it."""
    q = torch.arange(r0, r1, device=DEV)[:, None]
    k = torch.arange(k0, k1, device=DEV)[None, :]
    m = (k <= q)[None]
    if ds is not None:
        m = m & (k[None] >= ds[:, r0:r1, None].long())
    if window is not None:
        m = m & (k > q - window)[None]
    return m


def _chunks(B, S, nh, ds, window):
    """(r0, r1, k_lo): query-row chunks and the first key any of their rows can see."""
    R = max(128, (CHUNK_ELEMS // (B * nh * S)) // 128 * 128)
    first = ds[:, :].min(0).values.tolist() if ds is not None else None
    for r0 in range(0, S, R):
        k_lo = first[r0] if first is not None else 0
        if window is not None:
            k_lo = max(k_lo, r0 - window + 1)
        yield r0, min(S, r0 + R), max(0, k_lo)


def _heads(qkv, nh, nkv):
    """q, k, v in fp64 as [B, nh, S, d], k and v repeated over the GQA group."""
    g = nh // nkv
    x = qkv.double().permute(0, 2, 1, 3)
    return x[:, :nh], x[:, nh:nh + nkv].repeat_interleave(g, 1), x[:, nh + nkv:].repeat_interleave(g, 1)


# ------------------------------------------------------------------------------------------------------------------
# fp64 references
# ------------------------------------------------------------------------------------------------------------------
def _fwd64(qkv, nh, nkv, scale, ds=None, window=None):
    """Exact O and lse, the companion P |V|, the score term, the visible-key count n and the correctly rounded flash
    attention's O (P rounded to bf16 with the final row max).  Tensors are [B, nh, S, d] / [B, nh, S]."""
    B, S = qkv.shape[:2]
    q, k, v = _heads(qkv, nh, nkv)
    r = {name: torch.empty(B, nh, S, D, device=DEV, dtype=torch.float64) for name in ("o", "comp", "score", "yard")}
    r["lse"] = torch.empty(B, nh, S, device=DEV, dtype=torch.float64)
    r["n"] = torch.empty(B, 1, S, 1, device=DEV, dtype=torch.float64)
    c0 = D * U * scale
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
    their companions, score terms, the accumulation counts and the correctly rounded flash backward's gradients
    (P and dS rounded to bf16).  dQ tensors are [B, nh, S, d], dK / dV tensors [B, nkv, S, d]."""
    B, S = qkv.shape[:2]
    g = nh // nkv
    q, k, v = _heads(qkv, nh, nkv)
    dO = do.double().permute(0, 2, 1, 3)
    o64 = o.double().permute(0, 2, 1, 3)
    delta = (dO * o64).sum(-1, keepdim=True)
    dabs = (dO.abs() * o64.abs()).sum(-1, keepdim=True)
    lse = lse.double()[..., None]
    z = lambda: torch.zeros(B, nh, S, D, device=DEV, dtype=torch.float64)  # noqa: E731
    r = {name: z() for name in ("dq", "dq_comp", "dq_score", "dq_yard", "dk", "dk_comp", "dk_score", "dk_yard",
                                "dv", "dv_comp", "dv_score", "dv_yard")}
    nq = torch.zeros(B, 1, S, 1, device=DEV, dtype=torch.float64)
    nk = torch.zeros(B, 1, S, 1, device=DEV, dtype=torch.float64)
    c0 = D * U * scale
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
        out[name] = val if name.startswith("dq") else val.view(B, nkv, g, S, D).sum(2)
    for name in ("dq_yard", "dk_yard", "dv_yard"):
        out[name] = out[name].to(BF16)
    out["nq"], out["nk"] = nq, nk * g
    return out


# ------------------------------------------------------------------------------------------------------------------
# the two bounds
# ------------------------------------------------------------------------------------------------------------------
def _elem_c(got, exact, comp, score, n):
    """The least c the element bound needs; a NaN or an error the bound cannot cover at all gives inf.  An absolute
    2^-100 is allowed on top: the kernels' exp2 flushes p below fp32's normal range (2^-126) to zero."""
    num = (got.double() - exact).abs_().sub_(exact.abs() * 2.0 ** -8).sub_(comp * 2.0 ** -8).sub_(2.0 ** -100)
    den = (comp * (n * U)).add_(score)
    c = torch.where(num <= 0, torch.zeros_like(num), num / den)
    c = torch.where(torch.isnan(c), torch.full_like(c, float("inf")), c)
    return c.max().item()


def _lse_c(got, exact):
    err = (got.double() - exact).abs() / ((1 + exact.abs()) * 2.0 ** -23)
    return torch.where(torch.isnan(err), torch.full_like(err, float("inf")), err).max().item()


def _worst_tile(got, exact):
    """Largest relative L2 error over the (batch, head, 128-row tile) blocks of [B, H, S, d] tensors."""
    B, H, S, _ = exact.shape
    diff = (got.double() - exact).reshape(B, H, S // 128, -1).square().sum(-1)
    want = exact.reshape(B, H, S // 128, -1).square().sum(-1)
    rel = (diff / want.clamp_min(1e-300)).sqrt()
    return torch.where(torch.isnan(rel), torch.full_like(rel, float("inf")), rel).max().item()


def _check_tiles(tag, got, exact, yards):
    """``got`` against every yardstick in ``yards`` (name -> bf16 result of the same computation).  An output that is
    exactly zero (dQ, dK where every row sees only itself) has no relative error: the element bound judges it."""
    if not exact.abs().max().item() > 0:
        return ""
    tile = _worst_tile(got, exact)
    msg = []
    for name, y in yards.items():
        yt = _worst_tile(y, exact)
        msg.append(f"{name} {yt:.3e} ({tile / max(yt, 1e-30):.3f}x)")
        assert tile <= TILE_FACTOR * yt + TILE_SLACK, f"{tag}: worst tile {tile:.3e} vs {name} {yt:.3e}"
    return f"tile {tile:.3e} vs " + ", ".join(msg)


def _flash_sdpa(qkv, do, nh, nkv, scale):
    """PyTorch's bf16 flash attention (FA2) on the same inputs: O and dQ / dK / dV as [B, H, S, d].  The flash
    backend takes the GQA layout itself (``enable_gqa=True``), so dK / dV come back summed over the group."""
    x = qkv.detach().permute(0, 2, 1, 3)
    q, k, v = (t.contiguous().requires_grad_(True) for t in (x[:, :nh], x[:, nh:nh + nkv], x[:, nh + nkv:]))
    with sdpa_kernel(SDPBackend.FLASH_ATTENTION):
        o = torch.nn.functional.scaled_dot_product_attention(q, k, v, is_causal=True, scale=scale,
                                                             enable_gqa=nh != nkv)
        o.backward(do.permute(0, 2, 1, 3))
    return o.detach(), q.grad, k.grad, v.grad


# ------------------------------------------------------------------------------------------------------------------
# the kernels against fp64
# ------------------------------------------------------------------------------------------------------------------
# (B, S, nh, nkv, scale, pattern, documents, window)
CASES = {
    "one-tile": (1, 128, 1, 1, SC, "normal", None, None),
    "odd-tiles-b3": (3, 384, 4, 4, 0.05, "normal", None, None),
    "group16-sink": (2, 640, 16, 1, SC, "sink", None, None),
    "bench-4096": (1, 4096, 32, 8, SC, "normal", None, None),
    "70b-heads-peaked": (1, 2048, 64, 8, 1.0, "peaked", None, None),
    "16k-late-max": (1, 16384, 4, 1, SC, "late_max", None, None),
    "32k": (1, 32768, 2, 1, SC, "normal", None, None),
    "32k-w4096": (1, 32768, 2, 1, SC, "normal", None, 4096),
    "docs-offset-v": (2, 1024, 4, 2, SC, "offset_v", "edges", None),
    "docs-uniform": (2, 1024, 4, 1, 0.05, "uniform", "edges", None),
    "docs-late-max": (2, 2048, 4, 2, SC, "late_max", "edges", None),
    "one-token-docs": (2, 256, 4, 2, SC, "normal", "tokens", None),
    "w1": (2, 384, 4, 2, SC, "normal", None, 1),
    "w127-peaked": (1, 1024, 4, 1, SC, "peaked", None, 127),
    "w128-sink": (2, 512, 2, 2, SC, "sink", None, 128),
    "w129-offset-v": (1, 1024, 8, 2, 1.0, "offset_v", None, 129),
    "wS-1-uniform": (1, 512, 4, 4, SC, "uniform", None, 511),
    "docs-w129": (2, 1024, 4, 2, SC, "normal", "edges", 129),
    "docs-w127-late-max": (2, 2048, 4, 1, 0.05, "late_max", "edges", 127),
}


@pytest.mark.parametrize("case", list(CASES))
def test_kernels_against_fp64(case):
    B, S, nh, nkv, scale, pattern, layout, window = CASES[case]
    C = _C()
    qkv, do = _inputs(B, S, nh, nkv, pattern, scale, seed=len(case))
    ds = _docs(B, S, layout)
    plain = ds is None and window is None
    f = _fwd64(qkv, nh, nkv, scale, ds, window)
    sdpa = _flash_sdpa(qkv, do, nh, nkv, scale) if plain else None
    lines = []
    for version in (1, 2):
        o, lse = C.attn_fwd(qkv, nh, nkv, scale, version, doc_start=ds, window=window)
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
        g = C.attn_bwd(do, qkv, o_in, lse_in, nh, nkv, scale, None, mode, doc_start=ds, window=window)
        for i, name in enumerate(("dq", "dk", "dv")):
            got = g[:, :, sl[name]].permute(0, 2, 1, 3)
            n = b["nq"] if name == "dq" else b["nk"]
            c = _elem_c(got, b[name], b[name + "_comp"], b[name + "_score"], n)
            yards = {"rounded": b[name + "_yard"], **({"FA2": sdpa[1 + i]} if plain else {})}
            lines.append(f"bwd mode {mode} {name}: c {c:.3g}  "
                         f"{_check_tiles(f'{case} mode {mode} {name}', got, b[name], yards)}")
            assert c <= cmax[name], f"{case} mode {mode}: an element of {name} needs c = {c:.3g} > {cmax[name]}"
    print(f"\n{case}:\n  " + "\n  ".join(lines))


def test_attention_qkv_autograd_against_true_fp64_gradient():
    """Forward -> backward through autograd at Llama-2-7B (32:32) and Mistral-7B (32:8, W 4096) head geometry with
    the heads reduced to 4:4 and 4:1, against the true fp64 gradient (the backward formula on the exact O and lse),
    judged with the tile yardstick."""
    for tag, (S, nh, nkv, window) in {"llama-2-7b": (4096, 4, 4, None), "mistral-7b": (8192, 4, 1, 4096)}.items():
        qkv, do = _inputs(1, S, nh, nkv, "normal", SC, seed=9)
        x = qkv.clone().requires_grad_(True)
        out = ops.attention_qkv(x * 1.0, nh, nkv, window=window)
        out.backward(do)
        f = _fwd64(qkv, nh, nkv, SC, None, window)
        msg = [_check_tiles(f"{tag} O", out.permute(0, 2, 1, 3), f["o"], {"rounded": f["yard"]})]
        b = _bwd64(qkv, do, f["o"].permute(0, 2, 1, 3), f["lse"], nh, nkv, SC, None, window)
        for name, sl in (("dq", slice(0, nh)), ("dk", slice(nh, nh + nkv)), ("dv", slice(nh + nkv, None))):
            got = x.grad[:, :, sl].permute(0, 2, 1, 3)
            msg.append(f"{name} " + _check_tiles(f"{tag} {name}", got, b[name], {"rounded": b[name + "_yard"]}))
        print(f"\n{tag}: " + "; ".join(msg))


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
    o, lse = C.attn_fwd(qkv, SNH, SNKV, SC, version, doc_start=ds, window=window)
    g = C.attn_bwd(do, qkv, o, lse, SNH, SNKV, SC, None, mode, doc_start=ds, window=window)
    return o, lse, g


def _bits_equal(a, b):
    return torch.equal(a.view(torch.int16) if a.dtype == BF16 else a.view(torch.int32),
                       b.view(torch.int16) if b.dtype == BF16 else b.view(torch.int32))


def test_visibility_helper_is_the_reference_mask():
    for mask in MASKS:
        ds, window = _struct_mask(mask)
        want = ref.document_mask(ds, SS, window, device=DEV).expand(SB, SS, SS)
        assert torch.equal(_vis_all(ds, window), want), mask


@pytest.mark.parametrize("mask", list(MASKS))
def test_invisible_keys_and_queries_do_not_matter(mask):
    """Replacing K and V of key k0 leaves O, lse and dQ of every row that cannot see k0 unchanged, bit for bit;
    replacing Q and dO of query q0 leaves dK and dV of every key q0 cannot see unchanged.  Positions: the tile and
    half-tile edges, the last key, and keys just outside some row's document or window."""
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


def _block_any(vis, rb, cb):
    """[B, S/rb, S/cb]: some (row, column) pair of the block is visible."""
    B, R, Cn = vis.shape
    return vis.view(B, R // rb, rb, Cn // cb, cb).any(4).any(2)


@pytest.mark.parametrize("mask", list(MASKS))
def test_nan_reaches_exactly_the_outputs_that_depend_on_it(mask):
    """Forward: a NaN in one element of K (batch b, kv head h, key k) makes O and lse NaN exactly at (b, the q heads
    of h's group, the rows that see k).  Backward: a NaN in V of key k makes dK NaN at exactly (b, h, k) and leaves
    dV finite; a NaN in dO of query q makes dQ NaN at exactly (b, its head, q).  The gradient MMAs also multiply the
    masked entries of a processed block, where dS = 0 * (dP - delta) carries a NaN of dP on, so dQ (dK / dV) is
    asserted NaN where the dependence is real and finite only outside every block the kernel processes with the NaN:
    the 128-query x 64-key (128-key x 64-query) blocks with no visible pair."""
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
            o, lse = _C().attn_fwd(x, SNH, SNKV, SC, version, doc_start=ds, window=window)
            assert torch.equal(torch.isnan(o).any(-1), want), (mask, version, b, h, k)
            assert torch.equal(torch.isnan(o).all(-1), want), (mask, version, b, h, k)
            assert torch.equal(torch.isnan(lse), want.permute(0, 2, 1)), (mask, version, b, h, k)
            # backward, NaN in V
            o, lse = _C().attn_fwd(qkv, SNH, SNKV, SC, version, doc_start=ds, window=window)
            x = qkv.clone()
            x[b, k, SNH + SNKV + h, 5] = float("nan")
            gr = _C().attn_bwd(do, x, o, lse, SNH, SNKV, SC, None, mode, doc_start=ds, window=window)
            bad = torch.isnan(gr).any(-1)
            want_k = torch.zeros(SB, SS, SNKV, dtype=torch.bool, device=DEV)
            want_k[b, k, h] = True
            assert torch.equal(bad[:, :, SNH:SNH + SNKV], want_k), (mask, mode, "dK", b, h, k)
            assert not bad[:, :, SNH + SNKV:].any(), (mask, mode, "dV", b, h, k)
            dq_bad = bad[:, :, :SNH]
            assert torch.equal(dq_bad[:, :, ~heads], torch.zeros_like(dq_bad[:, :, ~heads])), (mask, mode, b, h, k)
            assert torch.equal(dq_bad[1 - b], torch.zeros_like(dq_bad[1 - b])), (mask, mode, b, h, k)
            assert dq_bad[b][vis[b, :, k]][:, heads].all(), (mask, mode, "dQ where real", b, h, k)
            seen = _block_any(vis[b:b + 1], 128, 64)[0, :, k // 64]            # [S/128]: blocks processed with k
            assert not dq_bad[b].view(SS // 128, 128, SNH)[~seen].any(), (mask, mode, "dQ outside", b, h, k)
            # backward, NaN in dO of query k (head hq)
            hq = h * g + 1
            d1 = do.clone()
            d1[b, k, hq, 9] = float("nan")
            gr = _C().attn_bwd(d1, qkv, o, lse, SNH, SNKV, SC, None, mode, doc_start=ds, window=window)
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


def _nan_padded(t):
    """``t`` as a contiguous view starting 16 bytes into a NaN-filled allocation that ends 16 bytes after it."""
    buf = torch.full((t.numel() + 16,), float("nan"), device=DEV, dtype=t.dtype)
    view = buf[8:8 + t.numel()].view(t.shape)
    view.copy_(t)
    return view


@pytest.mark.parametrize("mask", list(MASKS))
def test_reads_stay_inside_qkv_and_d_o(mask):
    """``qkv`` and ``d_o`` inside NaN-filled allocations: a read past either end would turn into NaN."""
    ds, window = _struct_mask(mask)
    qkv, do = _inputs(SB, SS, SNH, SNKV, "normal", SC, seed=41)
    pq, pd = _nan_padded(qkv), _nan_padded(do)
    for version, mode in ((1, 1), (1, 2), (2, 1), (2, 2)):
        o0, l0, g0 = _run(qkv, do, ds, window, version, mode)
        o1, l1, g1 = _run(pq, pd, ds, window, version, mode)
        assert torch.isfinite(o1).all() and torch.isfinite(g1).all(), (mask, version, mode)
        assert _bits_equal(o0, o1) and _bits_equal(l0, l1) and _bits_equal(g0, g1), (mask, version, mode)


@pytest.mark.parametrize("nh,nkv", [(4, 2), (4, 1), (16, 16)])
@pytest.mark.parametrize("how", ["w1", "one-token-docs", "one-token-docs+w1"])
def test_rows_that_see_only_themselves(how, nh, nkv):
    """With W = 1 or one-token documents, P = 1 on the diagonal and 0 elsewhere: O equals V bit for bit, and dV
    equals the fp32 sum of dO over the GQA group, rounded to bf16 once."""
    B, S = 2, 384
    ds = _docs(B, S, "tokens") if "docs" in how else None
    window = 1 if "w1" in how else None
    qkv, do = _inputs(B, S, nh, nkv, "normal", SC, seed=51)
    C = _C()
    v = qkv[:, :, nh + nkv:]
    dv = do.float().view(B, S, nkv, nh // nkv, D).sum(3).to(BF16)
    for version in (1, 2):
        o, lse = C.attn_fwd(qkv, nh, nkv, SC, version, doc_start=ds, window=window)
        assert _bits_equal(o, v.repeat_interleave(nh // nkv, 2).contiguous()), (how, version)
        for mode in (1, 2):
            g = C.attn_bwd(do, qkv, o, lse, nh, nkv, SC, None, mode, doc_start=ds, window=window)
            assert _bits_equal(g[:, :, nh + nkv:].contiguous(), dv), (how, version, mode)


# ------------------------------------------------------------------------------------------------------------------
# refused arguments
# ------------------------------------------------------------------------------------------------------------------
def _refused(call, match):
    torch.cuda.synchronize()
    n0 = _ext.launch_count()
    with pytest.raises(RuntimeError, match=match):
        call()
    assert _ext.launch_count() == n0, "a refused call launched a kernel"


def _misaligned(t, elems):
    """A contiguous copy of ``t`` that starts ``elems`` elements into its allocation."""
    buf = torch.zeros(t.numel() + 16, device=DEV, dtype=t.dtype)
    view = buf[elems:elems + t.numel()].view(t.shape)
    view.copy_(t)
    return view


def test_binding_refuses_bad_heads_and_scale():
    C = _C()
    S = 256
    for nh, nkv, match in ((0, 1, "nh and nkv"), (2, 0, "nh and nkv"), (-2, 2, "nh and nkv"), (6, 4, "multiple of nkv"),
                           (3, 2, "multiple of nkv")):
        qkv = torch.randn(1, S, max(nh + 2 * nkv, 1), D, device=DEV).to(BF16)
        do = torch.randn(1, S, max(nh, 1), D, device=DEV).to(BF16)
        o = torch.zeros_like(do)
        lse = torch.zeros(1, max(nh, 1), S, device=DEV)
        for version in (1, 2):
            _refused(lambda: C.attn_fwd(qkv, nh, nkv, SC, version), match)
        for mode in (1, 2):
            _refused(lambda: C.attn_bwd(do, qkv, o, lse, nh, nkv, SC, None, mode), match)
    nh, nkv = 2, 1
    qkv = torch.randn(1, S, 4, D, device=DEV).to(BF16)
    do = torch.randn(1, S, nh, D, device=DEV).to(BF16)
    o, lse = C.attn_fwd(qkv, nh, nkv, SC)
    # 1e-300 and 1e300 are finite and positive as doubles but 0 and inf in the kernels' fp32
    for bad in (0.0, -0.0, -SC, float("nan"), float("inf"), -float("inf"), 1e-300, 1e300):
        for version in (1, 2):
            _refused(lambda: C.attn_fwd(qkv, nh, nkv, bad, version), "scale")
        for mode in (1, 2):
            _refused(lambda: C.attn_bwd(do, qkv, o, lse, nh, nkv, bad, None, mode), "scale")
        if abs(bad) not in (1e-300, 1e300):
            n0 = _ext.launch_count()
            with pytest.raises(ValueError, match="scale"):
                ops.attention_qkv(qkv, nh, nkv, scale=bad)
            assert _ext.launch_count() == n0


def test_binding_refuses_bad_qkv_version_and_mode():
    C = _C()
    nh, nkv, S = 2, 1, 256
    qkv = torch.randn(1, S, 4, D, device=DEV).to(BF16)
    do = torch.randn(1, S, nh, D, device=DEV).to(BF16)
    o, lse = C.attn_fwd(qkv, nh, nkv, SC)
    for elems in (1, 4):   # 2 and 8 bytes past a 16-byte boundary
        bad = _misaligned(qkv, elems)
        _refused(lambda: C.attn_fwd(bad, nh, nkv, SC), "qkv must start on a 16-byte boundary")
        _refused(lambda: C.attn_bwd(do, bad, o, lse, nh, nkv, SC), "qkv must start on a 16-byte boundary")
    for bad in (torch.randn(1, 200, 4, D, device=DEV).to(BF16), torch.empty(1, 0, 4, D, device=DEV, dtype=BF16),
                torch.empty(0, S, 4, D, device=DEV, dtype=BF16)):
        _refused(lambda: C.attn_fwd(bad, nh, nkv, SC), "qkv must have B >= 1")
    for bad in (qkv.float(), qkv.cpu(), qkv.transpose(1, 2).contiguous().transpose(1, 2)):
        _refused(lambda: C.attn_fwd(bad, nh, nkv, SC), "qkv must be a contiguous bf16 CUDA tensor")
    _refused(lambda: C.attn_fwd(qkv[..., :64].contiguous(), nh, nkv, SC), r"qkv must be \[B, S")
    for version in (-1, 3):
        _refused(lambda: C.attn_fwd(qkv, nh, nkv, SC, version), "version")
    for mode in (-1, 3):
        _refused(lambda: C.attn_bwd(do, qkv, o, lse, nh, nkv, SC, None, mode), "mode")


def test_binding_refuses_bad_backward_tensors():
    C = _C()
    nh, nkv, S = 2, 1, 256
    qkv = torch.randn(2, S, 4, D, device=DEV).to(BF16)
    do = torch.randn(2, S, nh, D, device=DEV).to(BF16)
    o, lse = C.attn_fwd(qkv, nh, nkv, SC)
    bad_rows = [
        (lambda t: t.float(), "contiguous bf16"),
        (lambda t: t.transpose(1, 2).contiguous().transpose(1, 2), "contiguous bf16"),
        (lambda t: t[:1].contiguous(), r"\[B, S, nh, 128\]"),
        (lambda t: t[:, :128].contiguous(), r"\[B, S, nh, 128\]"),
        (lambda t: torch.cat([t, t], 2), r"\[B, S, nh, 128\]"),
        (lambda t: t.reshape(2, S, nh * 2, 64), r"\[B, S, nh, 128\]"),
        (lambda t: t.cpu(), "device of qkv"),
        (lambda t: _misaligned(t, 1), "16-byte boundary"),
        (lambda t: _misaligned(t, 4), "16-byte boundary"),
    ]
    for mode in (1, 2):
        for make, match in bad_rows:
            bad = make(o)
            _refused(lambda: C.attn_bwd(do, qkv, bad, lse, nh, nkv, SC, None, mode), r"(?<!\w)o must.*" + match)
            bad = make(do)
            _refused(lambda: C.attn_bwd(bad, qkv, o, lse, nh, nkv, SC, None, mode), "d_o must.*" + match)
        for bad, match in ((lse.double(), "lse must be a contiguous fp32"), (lse.transpose(1, 2).contiguous()
                           .transpose(1, 2), "lse must be a contiguous fp32"), (lse[:, :1].contiguous(), r"lse must be \[B, nh, S\]"),
                           (lse[..., :128].contiguous(), r"lse must be \[B, nh, S\]"),
                           (lse.reshape(2, nh * S), r"lse must be \[B, nh, S\]"), (lse.cpu(), "lse must be on the device")):
            _refused(lambda: C.attn_bwd(do, qkv, o, bad, nh, nkv, SC, None, mode), match)
        for bad in (torch.zeros(1024, dtype=torch.int32, device=DEV), torch.zeros(512, dtype=torch.long, device=DEV),
                    torch.zeros(1024, dtype=torch.long), torch.zeros(2048, dtype=torch.long, device=DEV)[::2]):
            _refused(lambda: C.attn_bwd(do, qkv, o, lse, nh, nkv, SC, bad, mode), "trace")
