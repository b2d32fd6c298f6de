"""Tensor-parallel fused kernels (AG->GEMM, GEMM->RS, K-gathered wgrad, vocab-parallel CE, hidden-parallel
embedding) on 2 GPUs vs a single-GPU run with the same seed and batch.

The numerics of the tensor-parallel and FSDP engines at world size 1 (loss, every gradient as AdamW consumed it and
the update, against an fp32 model) are checked on one GPU by ``test_gpu_engines_reference.py``; this file remains
the check over real NVLink."""
import pytest
import torch

from dist_utils import run_distributed

pytestmark = [pytest.mark.gpu, pytest.mark.multigpu]


def _gemm_modes(rank, world):
    """Each distributed GEMM mode against torch.distributed + matmul."""
    import torch.distributed as dist

    from distributed_training_guide_b200 import _ext
    from distributed_training_guide_b200.parallel import bootstrap
    from distributed_training_guide_b200.parallel.symm import SymmGroup

    env = bootstrap.init_distributed("cuda")
    dev, C = env.device, _ext.load(True)
    sg = SymmGroup(dev)
    t = world
    Tl, H, n = 256, 512, 384
    T = Tl * t
    torch.manual_seed(10 + rank)
    out = {}
    # mode 1: all-gather(M) -> GEMM
    xs = sg.alloc(Tl * H, torch.bfloat16)
    x_local = torch.randn(Tl, H, device=dev).to(torch.bfloat16)
    xs.local.view(Tl, H).copy_(x_local)
    w = (0.05 * torch.randn(n, H, device=dev)).to(torch.bfloat16)
    parts = [torch.empty_like(x_local) for _ in range(t)]
    dist.all_gather(parts, x_local)
    x_full = torch.cat(parts)
    torch.cuda.synchronize(); dist.barrier()
    y = torch.empty(T, n, device=dev, dtype=torch.bfloat16)
    sg.barrier_()
    C.gemm_dist(1, xs.ptrs, [w.data_ptr()], [y.data_ptr()], T, n, H, H, H, n, True, False, t, rank, Tl)
    torch.cuda.synchronize()
    want = x_full.float() @ w.float().t()
    out["ag_gemm"] = ((y.float() - want).abs().max() / want.abs().max()).item()
    # mode 2: GEMM -> reduce-scatter push, then reduce
    a = torch.randn(T, n, device=dev).to(torch.bfloat16)
    w2 = (0.05 * torch.randn(H, n, device=dev)).to(torch.bfloat16)
    st = sg.alloc(t * Tl * H, torch.bfloat16)
    torch.cuda.synchronize(); dist.barrier()
    C.gemm_dist(2, [a.data_ptr()], [w2.data_ptr()], [p + rank * Tl * H * 2 for p in st.ptrs], T, H, n, n, n, H, True, False,
                t, rank, Tl)
    sg.barrier_()
    red = torch.empty(Tl, H, device=dev, dtype=torch.bfloat16)
    C.tp_reduce_parts(st.local.view(t, Tl, H), None, red)
    torch.cuda.synchronize()
    full = a.float() @ w2.float().t()
    dist.all_reduce(full)
    want = full[rank * Tl:(rank + 1) * Tl]
    out["gemm_rs"] = ((red.float() - want).abs().max() / want.abs().max()).item()
    # mode 3: wgrad with B gathered along K: dW[n, H] = dy^T[n, T] @ x_full[T, H]
    dy = torch.randn(T, n, device=dev).to(torch.bfloat16)
    dw = torch.empty(n, H, device=dev, dtype=torch.bfloat16)
    C.gemm_dist(3, [dy.data_ptr()], xs.ptrs, [dw.data_ptr()], n, H, T, n, H, H, False, False, t, rank, Tl)
    torch.cuda.synchronize()
    want = dy.float().t() @ x_full.float()
    out["wgrad_b"] = ((dw.float() - want).abs().max() / want.abs().max()).item()
    # mode 4: wgrad with A gathered along K: dW[H, n] = x_full^T[H, T] @ a[T, n]
    dw2 = torch.empty(H, n, device=dev, dtype=torch.bfloat16)
    C.gemm_dist(4, xs.ptrs, [a.data_ptr()], [dw2.data_ptr()], H, n, T, H, n, n, False, False, t, rank, Tl)
    torch.cuda.synchronize()
    want = x_full.float().t() @ a.float()
    out["wgrad_a"] = ((dw2.float() - want).abs().max() / want.abs().max()).item()
    # in-kernel all-gather by communication CTAs (bulk copies over NVLink + per-tile flags) -> GEMM
    Tl2, H2, n2 = 512, 1024, 768            # two 256-row tiles per rank, 32 KB pieces
    T2 = Tl2 * t
    ag = sg.alloc(T2 * H2, torch.bfloat16)
    full = ag.local.view(T2, H2)
    full.zero_()
    xl = torch.randn(Tl2, H2, device=dev).to(torch.bfloat16)
    full[rank * Tl2:(rank + 1) * Tl2].copy_(xl)
    parts = [torch.empty_like(xl) for _ in range(t)]
    dist.all_gather(parts, xl)
    xf = torch.cat(parts)
    flags = torch.zeros(T2 // 256, dtype=torch.int32, device=dev)
    for ep, (wm, bk) in enumerate([((0.05 * torch.randn(n2, H2, device=dev)).to(torch.bfloat16), True),
                                   ((0.05 * torch.randn(H2, n2, device=dev)).to(torch.bfloat16), False)], start=1):
        if ep == 2:  # second call: fresh data in my rows, stale gathered rows must be re-fetched
            xl = torch.randn(Tl2, H2, device=dev).to(torch.bfloat16)
            torch.cuda.synchronize(); dist.barrier()
            full[rank * Tl2:(rank + 1) * Tl2].copy_(xl)
            dist.all_gather(parts, xl)
            xf = torch.cat(parts)
        y2 = torch.empty(T2, n2, device=dev, dtype=torch.bfloat16)
        torch.cuda.synchronize(); dist.barrier()
        C.gemm_ag(ag.ptrs, wm, y2, bk, rank, Tl2, flags, ep, sg.pad_ptrs, sg._epochs(1), 2)
        torch.cuda.synchronize()
        want = xf.float() @ (wm.float().t() if bk else wm.float())
        out[f"gemm_ag_{ep}"] = ((y2.float() - want).abs().max() / want.abs().max()).item()
        out[f"gathered_copy_{ep}"] = (full.float() - xf.float()).abs().max().item()
    sg.check()
    return out


def test_distributed_gemm_modes():
    res = run_distributed(_gemm_modes, world=2, timeout=300)
    print(res[0])
    for r in res:
        for k, v in r.items():
            assert v < 2e-2, (k, v, r)


def _tp_train(rank, world, steps, parallelism, tp):
    from distributed_training_guide_b200.engine import TrainEngine

    torch.manual_seed(0)
    eng = TrainEngine.create("debug-llama-tp", parallelism=parallelism, batch_size=2, seq_length=256, lr=1e-3,
                             tensor_parallel=tp)
    losses = [float(eng.step(eng.synthetic_batch(seed=i))) for i in range(steps)]
    eng.close()
    return losses


def test_tensor_parallel_gpu_matches_single_gpu():
    from distributed_training_guide_b200.engine import TrainEngine

    steps = 3
    res = run_distributed(_tp_train, world=2, args=(steps, "tp", 2), timeout=300)
    torch.manual_seed(0)
    eng = TrainEngine.create("debug-llama-tp", parallelism="single", batch_size=2, seq_length=256, lr=1e-3, device="cuda")
    ref = [float(eng.step(eng.synthetic_batch(seed=i))) for i in range(steps)]
    for losses in res:
        for a, b in zip(losses, ref):
            assert abs(a - b) < 6e-2, (losses, ref)


def _fsdp_train(rank, world, steps, ckpt_act):
    from distributed_training_guide_b200.engine import TrainEngine

    torch.manual_seed(0)
    eng = TrainEngine.create("debug-llama-gqa", parallelism="fsdp", batch_size=2, seq_length=256, lr=1e-3,
                             checkpoint_activations=ckpt_act, num_layers=5)   # 5 layers over 3 rotating slots:
    # layers 0-1 are resharded after forward, so backward gathers them again
    e = eng.strategy.engine
    losses = [float(eng.step(eng.synthetic_batch(seed=i))) for i in range(steps)]
    sd = {k: v.float().cpu() for k, v in e.full_state_dict().items()}
    eng.close()
    return losses, sd


@pytest.mark.parametrize("ckpt_act", [False, True])
def test_fsdp_gpu_matches_single_gpu(ckpt_act):
    """FSDP on 2 GPUs (copy-engine unshard) vs one GPU on the concatenated batch: losses and the final weights."""
    from distributed_training_guide_b200.engine import TrainEngine

    steps, world = 3, 2
    res = run_distributed(_fsdp_train, world=world, args=(steps, ckpt_act), timeout=300)
    torch.manual_seed(0)
    eng = TrainEngine.create("debug-llama-gqa", parallelism="single", batch_size=2, seq_length=256, lr=1e-3, device="cuda",
                             num_layers=5)
    ref = []
    for i in range(steps):
        parts = []
        for r in range(world):
            g = torch.Generator().manual_seed(1000 * i + r)
            parts.append(torch.randint(0, eng.config.vocab_size, (2, 256), generator=g))
        ids = torch.cat(parts)
        ref.append(float(eng.step({"input_ids": ids, "labels": ids.clone()})))
    ref_sd = {k: v.detach().float().cpu() for k, v in eng.model.state_dict().items()}
    (l0, sd0), (l1, sd1) = res
    for i in range(steps):
        assert abs(0.5 * (l0[i] + l1[i]) - ref[i]) < 6e-2, (i, l0, l1, ref)
    import numpy as np

    for k in sd0:
        assert np.array_equal(sd0[k], sd1[k]), k
        assert np.abs(sd0[k] - ref_sd[k].numpy()).max() < 3e-2, k
