"""FSDP unshard fused into the consuming GEMM (gemm_wgmma.cu, B_MODE 3): the weight lives in the ranks' flat shards,
warp 1 of every CTA gathers it into the local full buffer while the tensor cores consume the rows that have arrived.
Checked against a plain fp32 matmul of the full weight, forward (B K-major) and dgrad (B MN-major) — needs >= 2 GPUs."""
import pytest
import torch

from dist_utils import run_distributed

pytestmark = [pytest.mark.gpu, pytest.mark.multigpu]


def _world():
    n = torch.cuda.device_count()
    return 2 if n < 4 else (4 if n < 8 else 8)


def _check(rank, world):
    import torch.distributed as dist

    from distributed_training_guide_b200.parallel import bootstrap
    from distributed_training_guide_b200.parallel.symm import SymmGroup

    env = bootstrap.init_distributed("cuda")
    dev = env.device
    sg = SymmGroup(dev)
    C = sg.C
    shift = 15                                  # 32 KB chunks (2 pieces each)
    N1, K1 = 1024, 512                          # forward weight  W1[N1, K1]  (y = x @ W1^T)
    R2, C2 = 768, 512                           # dgrad weight    W2[R2, C2]  (dx = dy @ W2), gathered along its rows
    n1, n2 = N1 * K1, R2 * C2
    total = n1 + n2
    per = total // world
    assert (per * 2) % (1 << shift) == 0 and (n1 * 2) % (1 << shift) == 0
    torch.manual_seed(1)
    flat = (torch.randn(total, device=dev) * 0.05).to(torch.bfloat16)      # identical on every rank
    shard = sg.alloc(per, torch.bfloat16)
    shard.local.copy_(flat[rank * per:(rank + 1) * per])
    full = torch.zeros(total, device=dev, dtype=torch.bfloat16)
    counters = torch.zeros(max(64, (total * 2) >> shift), device=dev, dtype=torch.int32)
    M = 512
    torch.manual_seed(10 + rank)
    x = torch.randn(M, K1, device=dev).to(torch.bfloat16)
    dy = torch.randn(M, R2, device=dev).to(torch.bfloat16)
    torch.cuda.synchronize()
    dist.barrier()
    out = {}
    ppc = (1 << shift) // 16384
    for gen in (1, 2):                          # two generations: counters are monotonic
        full.zero_()
        full[rank * per:(rank + 1) * per].copy_(shard.local)   # the local slice is the caller's job (a D2D copy)
        y = torch.empty(M, N1, device=dev, dtype=torch.bfloat16)
        C.gemm_bgather(x, full, y, True, N1, K1, shard.ptrs, per, 0, n1, counters, gen * ppc, shift, sg.pad_ptrs, rank,
                       sg._epochs(1))
        dx = torch.empty(M, C2, device=dev, dtype=torch.bfloat16)
        C.gemm_bgather(dy, full, dx, False, R2, C2, shard.ptrs, per, n1, n2, counters, gen * ppc, shift, sg.pad_ptrs,
                       rank, sg._epochs(1))
        torch.cuda.synchronize()
        w1 = flat[:n1].view(N1, K1).float()
        w2 = flat[n1:].view(R2, C2).float()
        out[f"gathered_{gen}"] = bool(torch.equal(full, flat))
        out[f"fwd_err_{gen}"] = ((y.float() - x.float() @ w1.t()).abs().max() / (x.float() @ w1.t()).abs().max()).item()
        out[f"dgrad_err_{gen}"] = ((dx.float() - dy.float() @ w2).abs().max() / (dy.float() @ w2).abs().max()).item()
        dist.barrier()
    sg.check()
    return out


def test_gemm_with_fused_fsdp_gather():
    res = run_distributed(_check, world=_world(), timeout=300)
    print(res[0])
    for r in res:
        for gen in (1, 2):
            assert r[f"gathered_{gen}"], r
            assert r[f"fwd_err_{gen}"] < 2e-2 and r[f"dgrad_err_{gen}"] < 2e-2, r
