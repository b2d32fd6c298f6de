"""wgmma flash-attention forward/backward vs an fp32 reference (causal, GQA, head_dim 128)."""
import math

import pytest
import torch

from distributed_training_guide_b200 import _ext, ops
from distributed_training_guide_b200.ops import reference as ref

pytestmark = pytest.mark.gpu
DEV = "cuda"


# Worst (batch, head, 128-row tile) relative error allowed for random-normal inputs.  Measured on an H100 at the
# shapes below: at most 2.4e-3 for O and 2.9e-3 for dQ / dK / dV, in both forward versions and backward modes.
FWD_TILE_TOL, GRAD_TILE_TOL, LSE_TOL = 8e-3, 1e-2, 1e-3


def _assert_tiles(name, got, want, tol, tile=128):
    """Relative error of every (batch, head, 128-row tile) block of two [B, S, heads, d] tensors, asserted on the
    worst block.  One norm over the whole output would hide a wrong slice of one head: at S 4096 with 32 heads a
    block is 1/1024 of the tensor.  Rows are queries for O and dQ, keys for dK and dV."""
    B, S, H, d = want.shape
    diff = (got.float() - want.float()).reshape(B, S // tile, tile, H, d).square().sum((2, 4))
    ref2 = want.float().reshape(B, S // tile, tile, H, d).square().sum((2, 4))
    rel = (diff / ref2.clamp_min(1e-30)).sqrt()
    b, t, h = (int(i) for i in torch.unravel_index(rel.argmax(), rel.shape))
    worst, whole = rel.max().item(), (diff.sum() / ref2.sum()).sqrt().item()
    assert worst < tol, (f"{name}: batch {b} head {h} rows {t * tile}..{t * tile + tile - 1}: rel {worst:.4g} "
                         f"(whole tensor {whole:.4g})")


def _ref_lse(qkv, nh, nkv, scale, chunk=512):
    """fp32 logsumexp of the causal scores [B, nh, S], a chunk of query rows at a time (S 4096 in one piece would
    need [B, nh, S, S] fp32)."""
    B, S = qkv.shape[:2]
    q = qkv[:, :, :nh].float().permute(0, 2, 1, 3)
    k = qkv[:, :, nh:nh + nkv].float().permute(0, 2, 1, 3).repeat_interleave(nh // nkv, 1)
    cols = torch.arange(S, device=qkv.device)
    out = torch.empty(B, nh, S, device=qkv.device)
    for r0 in range(0, S, chunk):
        rows = cols[r0:r0 + chunk]
        s = (q[:, :, r0:r0 + chunk] @ k.transpose(-1, -2)) * scale
        out[:, :, r0:r0 + chunk] = torch.logsumexp(s.masked_fill(cols[None, :] > rows[:, None], float("-inf")), -1)
    return out


def _ref_fwd_bwd(qkv, do, nh, nkv, scale):
    """fp32 reference output and d(qkv) for the upstream gradient ``do``."""
    qf = qkv.detach().float().requires_grad_(True)
    want = ref.attention(qf[:, :, :nh], qf[:, :, nh:nh + nkv], qf[:, :, nh + nkv:], causal=True, scale=scale)
    want.backward(do.float())
    return want.detach(), qf.grad


def _grad_slices(nh, nkv):
    return ("dq", slice(0, nh)), ("dk", slice(nh, nh + nkv)), ("dv", slice(nh + nkv, nh + 2 * nkv))


@pytest.mark.parametrize("version", [1, 2])
@pytest.mark.parametrize("B,S,nh,nkv", [(1, 128, 1, 1), (1, 256, 2, 1), (2, 384, 4, 2), (1, 1024, 8, 2), (1, 2048, 4, 4),
                                        (1, 4096, 32, 4), (2, 640, 8, 1)])
def test_attention_forward_versions(B, S, nh, nkv, version):
    """Both forward kernels (1: P through shared memory; 2: P kept in registers) against fp32 —
    including the bench shape (S 4096, 32 heads, GQA 8:1) and odd numbers of 128-row tiles (384, 640)."""
    torch.manual_seed(0)
    C = _ext.load(True)
    d = 128
    qkv = torch.randn(B, S, nh + 2 * nkv, d, device=DEV, dtype=torch.bfloat16)
    o, lse = C.attn_fwd(qkv, nh, nkv, 1.0 / math.sqrt(d), version)
    qf = qkv.float()
    want = ref.attention(qf[:, :, :nh], qf[:, :, nh:nh + nkv], qf[:, :, nh + nkv:], causal=True)
    _assert_tiles(f"forward v{version}", o, want, FWD_TILE_TOL)
    err = (lse - _ref_lse(qkv, nh, nkv, 1.0 / math.sqrt(d))).abs().max().item()
    assert err < LSE_TOL, f"forward v{version}: lse max err {err:.4g}"


@pytest.mark.parametrize("version", [1, 2])
def test_attention_forward_row_max_jumps_late(version):
    """Scores whose row maximum grows by far more than the lazy-rescale threshold in LATE key blocks, for SOME rows of
    a warp only (the rescale decision is per row, made by the four threads of a quad;
    random-normal inputs never take that branch after the first block)."""
    torch.manual_seed(3)
    C = _ext.load(True)
    B, S, nh, nkv, d = 1, 1024, 4, 2, 128
    qkv = torch.randn(B, S, nh + 2 * nkv, d, device=DEV, dtype=torch.bfloat16)
    boost = torch.ones(S, device=DEV)
    boost[300:310] = 5.0
    boost[700:] = 9.0                         # late keys dominate
    rows = torch.ones(S, device=DEV)
    rows[::3] = 0.05                          # every third query barely reacts: its max does not move
    qkv[:, :, nh:nh + nkv] *= boost[None, :, None, None].to(qkv.dtype)
    qkv[:, :, :nh] *= rows[None, :, None, None].to(qkv.dtype)
    o, lse = C.attn_fwd(qkv, nh, nkv, 1.0 / math.sqrt(d), version)
    torch.cuda.synchronize()
    qf = qkv.float()
    want = ref.attention(qf[:, :, :nh], qf[:, :, nh:nh + nkv], qf[:, :, nh + nkv:], causal=True)
    _assert_tiles(f"forward v{version}", o, want, 2e-2)   # strongly peaked scores: outside the measurement above


@pytest.mark.parametrize("B,S,nh,nkv", [(1, 128, 1, 1), (2, 256, 4, 2), (1, 1024, 8, 2), (1, 512, 4, 4), (1, 2048, 2, 1),
                                        (1, 4096, 8, 1), (1, 384, 2, 2)])
def test_attention_fwd_bwd(B, S, nh, nkv):
    torch.manual_seed(0)
    d = 128
    qkv = torch.randn(B, S, nh + 2 * nkv, d, device=DEV, dtype=torch.bfloat16, requires_grad=True)
    do = torch.randn(B, S, nh, d, device=DEV, dtype=torch.bfloat16)
    out = ops.attention_qkv(qkv * 1.0, nh, nkv)
    out.backward(do)
    want, gw = _ref_fwd_bwd(qkv, do, nh, nkv, 1.0 / math.sqrt(d))
    _assert_tiles("forward", out, want, FWD_TILE_TOL)
    for name, sl in _grad_slices(nh, nkv):
        _assert_tiles(name, qkv.grad[:, :, sl], gw[:, :, sl], GRAD_TILE_TOL)


@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("B,S,nh,nkv", [(1, 256, 2, 1), (1, 1024, 8, 2), (1, 2048, 4, 4), (2, 384, 4, 2)])
def test_attention_backward_modes(B, S, nh, nkv, mode):
    """Backward with P / dS staged through shared memory (mode 1) and kept in registers (mode 2, RS-form gradient
    MMAs) against the fp32 reference."""
    torch.manual_seed(0)
    C = _ext.load(True)
    d = 128
    sc = 1.0 / math.sqrt(d)
    qkv = torch.randn(B, S, nh + 2 * nkv, d, device=DEV, dtype=torch.bfloat16)
    do = torch.randn(B, S, nh, d, device=DEV, dtype=torch.bfloat16)
    o, lse = C.attn_fwd(qkv, nh, nkv, sc, 1)
    g = C.attn_bwd(do, qkv, o, lse, nh, nkv, sc, None, mode)
    _, gw = _ref_fwd_bwd(qkv, do, nh, nkv, sc)
    for name, sl in _grad_slices(nh, nkv):
        _assert_tiles(f"mode {mode} {name}", g[:, :, sl], gw[:, :, sl], GRAD_TILE_TOL)


def test_attention_lse():
    torch.manual_seed(1)
    C = _ext.load(True)
    B, S, nh, nkv, d = 1, 256, 2, 1, 128
    qkv = torch.randn(B, S, nh + 2 * nkv, d, device=DEV, dtype=torch.bfloat16)
    o, lse = C.attn_fwd(qkv, nh, nkv, 1.0 / math.sqrt(d))
    q = qkv[:, :, :nh].float().permute(0, 2, 1, 3)
    k = qkv[:, :, nh:nh + nkv].float().permute(0, 2, 1, 3).repeat_interleave(nh // nkv, 1)
    s = (q @ k.transpose(-1, -2)) / math.sqrt(d)
    s = s.masked_fill(~torch.ones(S, S, dtype=torch.bool, device=DEV).tril(), float("-inf"))
    want = torch.logsumexp(s, dim=-1)
    assert (lse - want).abs().max().item() < LSE_TOL


@pytest.mark.parametrize("mode", [1, 2])
def test_attention_softmax_scale(mode):
    """A softmax scale other than 1/sqrt(128): forward (version ``mode``), LSE and backward (mode ``mode``)."""
    torch.manual_seed(2)
    C = _ext.load(True)
    B, S, nh, nkv, d, sc = 2, 512, 4, 2, 128, 0.05
    qkv = torch.randn(B, S, nh + 2 * nkv, d, device=DEV, dtype=torch.bfloat16)
    do = torch.randn(B, S, nh, d, device=DEV, dtype=torch.bfloat16)
    o, lse = C.attn_fwd(qkv, nh, nkv, sc, mode)
    g = C.attn_bwd(do, qkv, o, lse, nh, nkv, sc, None, mode)
    want, gw = _ref_fwd_bwd(qkv, do, nh, nkv, sc)
    _assert_tiles("forward", o, want, FWD_TILE_TOL)
    err = (lse - _ref_lse(qkv, nh, nkv, sc)).abs().max().item()
    assert err < LSE_TOL, f"lse max err {err:.4g}"
    for name, sl in _grad_slices(nh, nkv):
        _assert_tiles(name, g[:, :, sl], gw[:, :, sl], GRAD_TILE_TOL)


@pytest.mark.parametrize("B,S,nh,nkv", [(2, 640, 8, 1), (1, 2048, 8, 2)])
def test_attention_deterministic(B, S, nh, nkv):
    """Both forward versions and both backward modes give bit-identical results on a second call (the backward
    sums dK / dV and dQ in fixed order: no atomics)."""
    torch.manual_seed(4)
    C = _ext.load(True)
    sc = 1.0 / math.sqrt(128)
    qkv = torch.randn(B, S, nh + 2 * nkv, 128, device=DEV, dtype=torch.bfloat16)
    do = torch.randn(B, S, nh, 128, device=DEV, dtype=torch.bfloat16)
    for version in (1, 2):
        (o1, l1), (o2, l2) = C.attn_fwd(qkv, nh, nkv, sc, version), C.attn_fwd(qkv, nh, nkv, sc, version)
        assert torch.equal(o1, o2) and torch.equal(l1, l2), f"forward v{version} differs between two calls"
    o, lse = C.attn_fwd(qkv, nh, nkv, sc, 1)
    for mode in (1, 2):
        g1 = C.attn_bwd(do, qkv, o, lse, nh, nkv, sc, None, mode)
        g2 = C.attn_bwd(do, qkv, o, lse, nh, nkv, sc, None, mode)
        assert torch.equal(g1, g2), f"backward mode {mode} differs between two calls"
