"""wgmma flash-attention forward/backward vs an fp32 reference (causal, GQA, head_dim 128)."""
import math

import pytest
import torch

from distributed_training_guide_b200 import _ext, ops
from distributed_training_guide_b200.ops import reference as ref

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _rel(a, b):
    a, b = a.float(), b.float()
    return ((a - b).norm() / (b.norm() + 1e-12)).item(), (a - b).abs().max().item()


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
    rel, mx = _rel(o, want)
    assert rel < 2e-2, f"forward v{version}: rel {rel:.4g} max {mx:.4g}"
    q = qf[:, :, :nh].permute(0, 2, 1, 3)
    k = qf[:, :, nh:nh + nkv].permute(0, 2, 1, 3).repeat_interleave(nh // nkv, 1)
    if S <= 2048:
        sc = (q @ k.transpose(-1, -2)) / math.sqrt(d)
        sc = sc.masked_fill(~torch.ones(S, S, dtype=torch.bool, device=DEV).tril(), float("-inf"))
        assert (lse - torch.logsumexp(sc, dim=-1)).abs().max().item() < 2e-2


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
    rel, mx = _rel(o, want)
    assert rel < 2e-2, f"forward v{version}: rel {rel:.4g} max {mx:.4g}"


@pytest.mark.parametrize("B,S,nh,nkv", [(1, 128, 1, 1), (2, 256, 4, 2), (1, 1024, 8, 2), (1, 512, 4, 4), (1, 2048, 2, 1),
                                        (1, 4096, 8, 1), (1, 384, 2, 2)])
def test_attention_fwd_bwd(B, S, nh, nkv):
    torch.manual_seed(0)
    d = 128
    qkv = torch.randn(B, S, nh + 2 * nkv, d, device=DEV, dtype=torch.bfloat16, requires_grad=True)
    do = torch.randn(B, S, nh, d, device=DEV, dtype=torch.bfloat16)
    out = ops.attention_qkv(qkv * 1.0, nh, nkv)
    out.backward(do)
    qf = qkv.detach().float().requires_grad_(True)
    want = ref.attention(qf[:, :, :nh], qf[:, :, nh:nh + nkv], qf[:, :, nh + nkv:], causal=True)
    want.backward(do.float())
    rel, mx = _rel(out, want)
    assert rel < 2e-2, f"forward: rel {rel:.4g} max {mx:.4g}"
    g, gw = qkv.grad, qf.grad
    for name, sl in (("dq", slice(0, nh)), ("dk", slice(nh, nh + nkv)), ("dv", slice(nh + nkv, nh + 2 * nkv))):
        rel, mx = _rel(g[:, :, sl], gw[:, :, sl])
        assert rel < 3e-2, f"{name}: rel {rel:.4g} max {mx:.4g}"


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
    qf = qkv.float().requires_grad_(True)
    want = ref.attention(qf[:, :, :nh], qf[:, :, nh:nh + nkv], qf[:, :, nh + nkv:], causal=True)
    want.backward(do.float())
    for name, sl in (("dq", slice(0, nh)), ("dk", slice(nh, nh + nkv)), ("dv", slice(nh + nkv, nh + 2 * nkv))):
        rel, mx = _rel(g[:, :, sl], qf.grad[:, :, sl])
        assert rel < 3e-2, f"mode {mode} {name}: rel {rel:.4g} max {mx:.4g}"


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
    assert (lse - want).abs().max().item() < 2e-2
