"""NVLink symmetric-memory collectives vs torch.distributed (NCCL) results — needs >= 2 GPUs.

The numerics of the plain-DDP and FSDP engines at world size 1 (loss, every gradient as AdamW consumed it and the
update, against an fp32 model and bit for bit against the single-GPU engine) are checked on one GPU by
``test_gpu_engines_reference.py``; this file remains the check over real NVLink."""
import math

import pytest
import torch

from dist_utils import run_distributed

pytestmark = [pytest.mark.gpu, pytest.mark.multigpu]


def _world():
    return 2 if torch.cuda.device_count() < 4 else (4 if torch.cuda.device_count() < 8 else 8)


def _comm_checks(rank, world):
    import torch.distributed as dist

    from distributed_training_guide_b200.parallel import bootstrap
    from distributed_training_guide_b200.parallel.symm import SymmGroup

    env = bootstrap.init_distributed("cuda")
    dev = env.device
    sg = SymmGroup(dev)
    out = {}
    n = 8 * world * 12345
    torch.manual_seed(100 + rank)
    # ---- all-reduce with fused scale ------------------------------------------------------------
    buf = sg.alloc(n, torch.bfloat16)
    x = torch.randn(n, device=dev).to(torch.bfloat16)
    buf.local.copy_(x)
    want = x.float().clone()
    dist.all_reduce(want)
    want = want / world
    torch.cuda.synchronize()
    dist.barrier()
    sg.allreduce_scale_(buf, 0, n, 1.0 / world)
    torch.cuda.synchronize()
    out["allreduce_err"] = (buf.local.float() - want).abs().max().item()
    # ---- fused reduce-scatter + AdamW + all-gather (ZeRO-1 bucket kernel) -------------------------------
    g = sg.alloc(n, torch.bfloat16)
    p = sg.alloc(n, torch.bfloat16)
    torch.manual_seed(7)
    p0 = torch.randn(n, device=dev).to(torch.bfloat16)     # identical replicas
    p.local.copy_(p0)
    torch.manual_seed(200 + rank)
    gl = (0.01 * torch.randn(n, device=dev)).to(torch.bfloat16)
    g.local.copy_(gl)
    gsum = gl.float().clone()
    dist.all_reduce(gsum)
    gavg = gsum / world
    per = n // world
    m = torch.zeros(per, device=dev, dtype=torch.bfloat16)
    v = torch.zeros(per, device=dev, dtype=torch.bfloat16)
    torch.cuda.synchronize()
    dist.barrier()
    hyper = (1e-2, 0.9, 0.999, 1e-8, 1e-2)
    sg.rs_adamw_(g, p, None, m, v, True, 0, n, hyper, 1, 1.0 / world)
    torch.cuda.synchronize()
    dist.barrier()
    pr = torch.nn.Parameter(p0.float().clone())
    opt = torch.optim.AdamW([pr], lr=1e-2, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2)
    pr.grad = gavg
    opt.step()
    out["zero1_err"] = (p.local.float() - pr.data).abs().max().item()
    # replicas identical after the push
    chk = p.local.float().clone()
    dist.broadcast(chk, src=0)
    out["zero1_replica_diff"] = (chk - p.local.float()).abs().max().item()
    # ---- all-gather of shards ---------------------------------------------------------------------------
    sh = sg.alloc(per, torch.bfloat16)
    sh.local.copy_(torch.full((per,), float(rank + 1), device=dev, dtype=torch.bfloat16))
    full = torch.zeros(n, device=dev, dtype=torch.bfloat16)
    torch.cuda.synchronize()
    dist.barrier()
    sg.allgather_(sh, full, 0, per)
    torch.cuda.synchronize()
    exp = torch.cat([torch.full((per,), float(r + 1)) for r in range(world)]).to(dev)
    out["allgather_err"] = (full.float() - exp).abs().max().item()
    full.zero_()
    sg.allgather_(sh, full, 0, per, copy_engine=True)  # barrier kernel + peer copies on the copy engines
    torch.cuda.synchronize()
    out["allgather_ce_err"] = (full.float() - exp).abs().max().item()
    # ---- bandwidth of the fused kernels (device-timed) ------------------------------------------------------
    big = 8 * world * (1 << 22)  # 64 Mi elements at world=2 -> 128 MiB bf16
    bb = sg.alloc(big, torch.bfloat16)
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(2):
        sg.allreduce_scale_(bb, 0, big, 1.0)
    torch.cuda.synchronize(); dist.barrier()
    s.record()
    for _ in range(5):
        sg.allreduce_scale_(bb, 0, big, 1.0)
    e.record(); torch.cuda.synchronize()
    ms = s.elapsed_time(e) / 5
    out["allreduce_ms_%dMiB" % (big * 2 >> 20)] = ms
    out["allreduce_busbw_GBs"] = 2 * (world - 1) / world * big * 2 / ms / 1e6
    t = torch.empty(big, device=dev, dtype=torch.bfloat16)
    for _ in range(2):
        dist.all_reduce(t)
    torch.cuda.synchronize(); dist.barrier()
    s.record()
    for _ in range(5):
        dist.all_reduce(t)
    e.record(); torch.cuda.synchronize()
    out["nccl_allreduce_ms"] = s.elapsed_time(e) / 5
    sg.check()
    return out


def test_symmetric_collectives():
    world = _world()
    res = run_distributed(_comm_checks, world=world, timeout=300)
    print(res[0])
    for r in res:
        assert r["allreduce_err"] < 0.05, r
        assert r["zero1_err"] < 0.05, r
        assert r["zero1_replica_diff"] == 0.0, r
        assert r["allgather_err"] == 0.0 and r["allgather_ce_err"] == 0.0, r


def _ddp_train(rank, world, steps):
    from distributed_training_guide_b200.engine import TrainEngine

    torch.manual_seed(0)
    eng = TrainEngine.create("debug-llama-gqa", parallelism="ddp", batch_size=2, seq_length=256, lr=1e-3)
    losses = [float(eng.step(eng.synthetic_batch(seed=i))) for i in range(steps)]
    sd = {k: v.detach().float().cpu() for k, v in eng.model.state_dict().items()}
    eng.close()
    return losses, sd


def test_ddp_zero1_gpu_matches_single_gpu():
    from distributed_training_guide_b200.engine import TrainEngine

    world, steps = 2, 3
    res = run_distributed(_ddp_train, world=world, args=(steps,), timeout=300)
    torch.manual_seed(0)
    eng = TrainEngine.create("debug-llama-gqa", parallelism="single", batch_size=2, seq_length=256, lr=1e-3, device="cuda")
    ref = []
    for i in range(steps):
        parts = []
        for r in range(world):
            g = torch.Generator().manual_seed(1000 * i + r)
            parts.append(torch.randint(0, eng.config.vocab_size, (2, 256), generator=g))
        ids = torch.cat(parts)
        ref.append(float(eng.step({"input_ids": ids, "labels": ids.clone()})))
    (l0, sd0), (l1, sd1) = res
    import numpy as np

    for k in sd0:
        assert np.array_equal(sd0[k], sd1[k]), f"replicas diverged: {k}"
    for i in range(steps):
        assert abs(0.5 * (l0[i] + l1[i]) - ref[i]) < 5e-2, (i, l0[i], l1[i], ref[i])


def _nvls_checks(rank, world):
    """The same two checks as above through the NVSwitch-multicast kernels (comm_nvls.cu) on buffers from the own
    VMM arena (csrc/symm_vmm.cpp: cuMemCreate + cuMulticastCreate/BindMem), plus the in-switch reduce-scatter."""
    import os

    os.environ["DTG_NVLS_KERNELS"] = "1"
    import torch.distributed as dist

    from distributed_training_guide_b200.parallel import bootstrap
    from distributed_training_guide_b200.parallel.symm import SymmGroup

    env = bootstrap.init_distributed("cuda")
    dev = env.device
    sg = SymmGroup(dev)
    if not sg.multicast:
        return {"skipped": f"no NVSwitch multicast on this system (arena mode {sg.mode})"}
    assert sg.mode == "vmm" and sg.nvls and sg.pads.mc_ptr
    out = {"mode": sg.mode, "chunks": sg._n_chunks}
    n = 8 * world * 12345
    torch.manual_seed(100 + rank)
    buf = sg.alloc(n, torch.bfloat16)
    x = torch.randn(n, device=dev).to(torch.bfloat16)
    buf.local.copy_(x)
    want = x.float().clone()
    dist.all_reduce(want)
    want = want / world
    torch.cuda.synchronize()
    dist.barrier()
    sg.allreduce_scale_(buf, 0, n, 1.0 / world)
    torch.cuda.synchronize()
    out["allreduce_err"] = (buf.local.float() - want).abs().max().item()
    g = sg.alloc(n, torch.bfloat16)
    p = sg.alloc(n, torch.bfloat16)
    torch.manual_seed(7)
    p0 = torch.randn(n, device=dev).to(torch.bfloat16)
    p.local.copy_(p0)
    torch.manual_seed(200 + rank)
    gl = (0.01 * torch.randn(n, device=dev)).to(torch.bfloat16)
    g.local.copy_(gl)
    gsum = gl.float().clone()
    dist.all_reduce(gsum)
    per = n // world
    m = torch.zeros(per, device=dev, dtype=torch.bfloat16)
    v = torch.zeros(per, device=dev, dtype=torch.bfloat16)
    torch.cuda.synchronize()
    dist.barrier()
    sg.rs_adamw_(g, p, None, m, v, True, 0, n, (1e-2, 0.9, 0.999, 1e-8, 1e-2), 1, 1.0 / world)
    torch.cuda.synchronize()
    dist.barrier()
    pr = torch.nn.Parameter(p0.float().clone())
    opt = torch.optim.AdamW([pr], lr=1e-2, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2)
    pr.grad = gsum / world
    opt.step()
    out["zero1_err"] = (p.local.float() - pr.data).abs().max().item()
    chk = p.local.float().clone()
    dist.broadcast(chk, src=0)
    out["zero1_replica_diff"] = (chk - p.local.float()).abs().max().item()
    # ---- GEMM -> reduce-scatter, reduce half in the switch (fused_tp.cu: tp_reduce_mc) ------------------------------
    Tl, H = 256, 512
    part = sg.alloc(world * Tl * H, torch.bfloat16)
    torch.manual_seed(300 + rank)
    mine = torch.randn(world * Tl, H, device=dev).to(torch.bfloat16)
    part.local.copy_(mine.reshape(-1))
    res = torch.randn(Tl, H, device=dev).to(torch.bfloat16)
    tot = mine.float().clone()
    dist.all_reduce(tot)
    want_rows = tot[rank * Tl:(rank + 1) * Tl] + res.float()
    y = torch.empty(Tl, H, device=dev, dtype=torch.bfloat16)
    torch.cuda.synchronize()
    sg.C.tp_reduce_mc(part.mc_ptr + rank * Tl * H * 2, res, y, sg.pad_ptrs, rank, sg._epochs(1), sg.err)
    torch.cuda.synchronize()
    out["reduce_mc_err"] = ((y.float() - want_rows).abs().max() / want_rows.abs().max()).item()
    sg.check()
    return out


def test_nvls_collectives():
    world = _world()
    res = run_distributed(_nvls_checks, world=world, timeout=300)
    if "skipped" in res[0]:
        pytest.skip(res[0]["skipped"])
    print(res[0])
    for r in res:
        assert r["allreduce_err"] < 0.05, r
        assert r["zero1_err"] < 0.05, r
        assert r["zero1_replica_diff"] == 0.0, r
        assert r["reduce_mc_err"] < 0.02, r
