"""sm_90a elementwise / reduction kernels vs the fp32 PyTorch reference of the same op."""
import math

import pytest
import torch

from distributed_training_guide_b200 import _ext, ops
from distributed_training_guide_b200.ops import reference as ref

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _close(a, b, atol, rtol, name=""):
    a, b = a.float(), b.float()
    err = (a - b).abs()
    tol = atol + rtol * b.abs()
    bad = (err > tol).float().mean().item()
    assert bad < 1e-3, f"{name}: {bad:.4%} elements out of tolerance, max err {err.max().item():.4g}"


@pytest.mark.parametrize("T,H", [(64, 256), (300, 4096), (128, 8192), (32, 16384), (17, 1024)])
@pytest.mark.parametrize("with_res", [False, True])
def test_rmsnorm_fwd_bwd(T, H, with_res):
    torch.manual_seed(0)
    x = torch.randn(T, H, device=DEV, dtype=torch.bfloat16, requires_grad=True)
    r = torch.randn(T, H, device=DEV, dtype=torch.bfloat16, requires_grad=True) if with_res else None
    w = (1 + 0.1 * torch.randn(H, device=DEV)).to(torch.bfloat16).requires_grad_(True)
    dy = torch.randn(T, H, device=DEV, dtype=torch.bfloat16)
    dh = torch.randn(T, H, device=DEV, dtype=torch.bfloat16)
    if with_res:
        y, h = ops.add_rms_norm(x, r, w, 1e-5)
        (y.float() * dy.float()).sum().add((h.float() * dh.float()).sum()).backward()
    else:
        y = ops.rms_norm(x, w, 1e-5)
        (y.float() * dy.float()).sum().backward()
    xf = x.detach().float().requires_grad_(True)
    rf = r.detach().float().requires_grad_(True) if with_res else None
    wf = w.detach().float().requires_grad_(True)
    hf = xf + rf if with_res else xf
    if with_res:
        hf = hf + (hf.to(torch.bfloat16).float() - hf).detach()  # the residual stream is rounded to bf16
    yf = hf * torch.rsqrt(hf.pow(2).mean(-1, keepdim=True) + 1e-5) * wf
    loss = (yf * dy.float()).sum()
    if with_res:
        loss = loss + (hf * dh.float()).sum()
    loss.backward()
    _close(y, yf, 2e-2, 2e-2, "y")
    _close(x.grad, xf.grad, 3e-2, 3e-2, "dx")
    if with_res:
        _close(r.grad, rf.grad, 3e-2, 3e-2, "dr")
    _close(w.grad, wf.grad, 0.5 + 0.02 * math.sqrt(T), 3e-2, "dw")


@pytest.mark.parametrize("B,S,nh,nkv,d", [(2, 64, 4, 2, 128), (1, 256, 32, 8, 128), (1, 128, 2, 2, 64)])
@pytest.mark.parametrize("per_token", [False, True])
def test_rope_inplace(B, S, nh, nkv, d, per_token):
    torch.manual_seed(0)
    qkv = torch.randn(B, S, nh + 2 * nkv, d, device=DEV, dtype=torch.bfloat16)
    pos = torch.arange(S, device=DEV)
    if per_token:
        pos = pos[None].expand(B, S) + torch.arange(B, device=DEV)[:, None]
    cos, sin = ref.rope_tables(pos, d, 1e4)
    want = torch.cat([ref.rope_apply(qkv[:, :, :nh + nkv], cos, sin), qkv[:, :, nh + nkv:]], dim=2)
    g = qkv.clone().requires_grad_(True)
    out = ops.rope_qkv_(g * 1.0, cos, sin, nh + nkv)
    _close(out, want, 2e-2, 2e-2, "rope")
    dout = torch.randn_like(out)
    out.backward(dout.clone())  # the op rotates its incoming gradient in place (it owns it in the model)
    want_g = torch.cat([ref.rope_apply(dout[:, :, :nh + nkv], cos, sin, inverse=True), dout[:, :, nh + nkv:]], dim=2)
    _close(g.grad, want_g, 2e-2, 2e-2, "rope bwd")


@pytest.mark.parametrize("T,I", [(64, 512), (1000, 11008), (33, 1792)])
def test_swiglu(T, I):
    torch.manual_seed(0)
    gu = torch.randn(T, 2 * I, device=DEV, dtype=torch.bfloat16, requires_grad=True)
    dh = torch.randn(T, I, device=DEV, dtype=torch.bfloat16)
    h = ops.swiglu(gu)
    h.backward(dh)
    gf = gu.detach().float().requires_grad_(True)
    g, u = gf.chunk(2, -1)
    hf = torch.nn.functional.silu(g) * u
    hf.backward(dh.float())
    _close(h, hf, 2e-2, 2e-2, "swiglu")
    _close(gu.grad, gf.grad, 3e-2, 3e-2, "swiglu bwd")


@pytest.mark.parametrize("T,V", [(128, 1024), (512, 32000), (64, 128256)])
def test_cross_entropy(T, V):
    torch.manual_seed(0)
    logits = (2.0 * torch.randn(T, V, device=DEV)).to(torch.bfloat16).requires_grad_(True)
    tgt = torch.randint(0, V, (T,), device=DEV)
    tgt[::7] = -100
    lf = logits.detach().float().requires_grad_(True)
    want = torch.nn.functional.cross_entropy(lf, tgt, ignore_index=-100)
    want.backward()
    x = (logits * 1.0)
    x.retain_grad()
    loss = ops.cross_entropy(x, tgt)
    (loss * 1.0).backward()
    assert abs(loss.item() - want.item()) < 2e-3 * max(1.0, abs(want.item())), (loss.item(), want.item())
    _close(logits.grad * T, lf.grad * T, 2e-3, 3e-2, "dlogits")
    # non-unit upstream gradient
    logits.grad = None
    x = logits * 1.0
    (ops.cross_entropy(x, tgt) * 0.5).backward()
    _close(logits.grad * T, 0.5 * lf.grad * T, 2e-3, 3e-2, "dlogits*0.5")


@pytest.mark.parametrize("case", ["all_ignored", "first_and_last_column", "one_row", "std20"])
def test_cross_entropy_edges(case):
    """Edges against fp64, every element within tolerance (no outlier budget): no valid target at all (loss 0 and
    zero dlogits, not NaN), targets in the first and last column, a single row, logits with std 20."""
    T, V, std = {"all_ignored": (64, 1024, 2.0), "first_and_last_column": (128, 32000, 2.0),
                 "one_row": (1, 128256, 2.0), "std20": (256, 32000, 20.0)}[case]
    torch.manual_seed(0)
    logits = (std * torch.randn(T, V, device=DEV)).to(torch.bfloat16)
    tgt = torch.randint(0, V, (T,), device=DEV)
    if case == "all_ignored":
        tgt.fill_(-100)
    elif case == "first_and_last_column":
        tgt[0::2], tgt[1::2] = 0, V - 1
    n_valid = int((tgt != -100).sum())
    lf = logits.double().requires_grad_(True)
    want = torch.nn.functional.cross_entropy(lf, tgt, ignore_index=-100, reduction="sum") / max(n_valid, 1)
    want.backward()
    x = logits.clone().requires_grad_(True)
    loss = ops.cross_entropy(x * 1.0, tgt)   # the op overwrites its input with dlogits
    loss.backward()
    assert torch.isfinite(loss) and torch.isfinite(x.grad).all(), (loss.item(), case)
    assert abs(loss.item() - want.item()) <= 1e-4 * max(1.0, abs(want.item())), (loss.item(), want.item())
    err = (x.grad.double() - lf.grad).abs()
    tol = 1e-6 / max(n_valid, 1) + 8e-3 * lf.grad.abs()   # 8e-3: two bf16 ulps
    bad = err > tol
    assert not bad.any(), f"{case}: {int(bad.sum())} of {err.numel()} dlogits out of tolerance, max err {err.max():.3g}"
    if case == "all_ignored":
        assert loss.item() == 0.0 and int(torch.count_nonzero(x.grad)) == 0


@pytest.mark.parametrize("T,V,H", [(256, 1000, 256), (4096, 32000, 4096)])
def test_embedding(T, V, H):
    torch.manual_seed(0)
    w = torch.randn(V, H, device=DEV, dtype=torch.bfloat16, requires_grad=True)
    ids = torch.randint(0, V, (T,), device=DEV)
    ids[: T // 4] = 3  # heavy duplicates exercise the atomics
    out = ops.embedding(ids, w)
    assert torch.equal(out, w.detach()[ids])
    dout = torch.randn(T, H, device=DEV, dtype=torch.bfloat16)
    out.backward(dout)
    want = torch.zeros(V, H, device=DEV)
    want.index_add_(0, ids, dout.float())
    _close(w.grad, want, 0.25, 5e-2, "embedding bwd")


@pytest.mark.parametrize("n", [8 * 1000, 8 * 123457])
@pytest.mark.parametrize("state_dtype", [torch.bfloat16, torch.float32])
def test_adamw_flat(n, state_dtype):
    torch.manual_seed(0)
    C = _ext.load(True)
    p = torch.randn(n, device=DEV).to(torch.bfloat16)
    g = (0.01 * torch.randn(n, device=DEV)).to(torch.bfloat16)
    m = torch.zeros(n, device=DEV, dtype=state_dtype)
    v = torch.zeros(n, device=DEV, dtype=state_dtype)
    pr = torch.nn.Parameter(p.clone().float())
    opt = torch.optim.AdamW([pr], lr=1e-2, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2)
    for step in range(1, 4):
        C.adamw_flat(p, g, m, v, 1e-2, 0.9, 0.999, 1e-8, 1e-2, step, 1.0)
        pr.grad = g.float()
        opt.step()
        if state_dtype == torch.float32:
            pr.data = pr.data.to(torch.bfloat16).float()  # parameters are stored in bf16 each step
    tol = 2e-2 if state_dtype == torch.float32 else 6e-2
    _close(p, pr.data, tol, 2e-2, "adamw")


def test_embedding_backward_deterministic_mode():
    """--deterministic routes the embedding gradient through the sorted, atomics-free kernel: equal to the fp32
    reference and bit-identical across runs (heavily repeated ids make the atomic version order-dependent)."""
    from distributed_training_guide_b200 import ops

    torch.manual_seed(0)
    V, H, T = 512, 1024, 8192
    w = (torch.randn(V, H, device="cuda") * 0.02).to(torch.bfloat16).requires_grad_(True)
    ids = torch.randint(0, 16, (2, T // 2), device="cuda")     # 16 distinct ids: ~512 rows summed per table row
    dout = torch.randn(2, T // 2, H, device="cuda").to(torch.bfloat16)
    want = torch.zeros(V, H, device="cuda")
    want.index_add_(0, ids.reshape(-1), dout.reshape(-1, H).float())
    outs = []
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True, warn_only=True)
    try:
        for _ in range(3):
            w.grad = None
            ops.embedding(ids, w).backward(dout)
            outs.append(w.grad.clone())
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=True)
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2])
    err = (outs[0].float() - want).abs().max().item() / want.abs().max().item()
    assert err < 1e-2, err
