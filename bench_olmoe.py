"""OLMoE benchmark on one GPU: prints one JSON record.

  * the grouped expert GEMM (forward gate|up shape of OLMoE-1B-7B at S 4096, B 1: 64 experts, top-8, H 2048, 2I 2048):
    useful TFLOP/s (real rows only) and the share of rows that are 128-row segment padding, against one gemm_bf16
    launch per expert over the same rows and one dense GEMM over the same total rows;
  * GB/s of route, permute and combine at that shape;
  * device-timed tokens/s and peak memory of OLMoE-1B-7B training steps (single-GPU engine).

The kernel shapes come from ``--model``'s config (experts, top-k, hidden size, 2 x the expert intermediate size);
``--layers N`` trains the model truncated to its first N layers (a model too large for one GPU).

    python bench_olmoe.py [--seq 4096] [--steps 3] [--warmup 1] [--model NAME] [--layers N]
"""
import argparse
import json
import subprocess
import sys
import time

import torch


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name()


def _time(fn, iters=20):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters / 1e3


def kernels(T, E=64, k=8, H=2048, N=2048):
    from distributed_training_guide_b200 import _ext

    C = _ext.load(required=True)
    g = torch.Generator(device="cuda").manual_seed(0)
    lg = torch.randn(T, E, device="cuda", generator=g).to(torch.bfloat16)
    x = torch.randn(T, H, device="cuda", generator=g).to(torch.bfloat16)
    W = (torch.randn(E, N, H, device="cuda", generator=g) * 0.02).to(torch.bfloat16)
    p, idx, w, pos, seg, tiles, row_tok, counts = C.moe_route(lg, k)
    xp = C.moe_permute(x, row_tok, seg, k)
    R = xp.shape[0]
    out = torch.empty(R, N, device="cuda", dtype=torch.bfloat16)
    segs = seg.tolist()
    cnt = counts.tolist()
    used = segs[-1]
    flop = 2.0 * T * k * N * H
    t_grp = _time(lambda: C.gemm_grouped(0, xp, W, out, seg, tiles))

    def per_expert():
        for e in range(E):
            if cnt[e]:
                C.gemm(xp[segs[e]:segs[e] + cnt[e]], W[e], out[segs[e]:segs[e] + cnt[e]], False, True)
    t_loop = _time(per_expert)
    Wd = W[0]
    xd = xp[:T * k]
    outd = out[:T * k]
    t_dense = _time(lambda: C.gemm(xd, Wd, outd, False, True))
    t_route = _time(lambda: C.moe_route(lg, k))
    t_perm = _time(lambda: C.moe_permute(x, row_tok, seg, k))
    yp = torch.randn(R, H, device="cuda", generator=g).to(torch.bfloat16)
    t_comb = _time(lambda: C.moe_combine(yp, pos, w))
    route_bytes = T * E * 2 + T * E * 4 + T * k * 16 + R * 4
    move_bytes = (T * H + used * H) * 2            # read tokens, write permuted rows
    comb_bytes = (T * k * H + T * H) * 2 + T * k * 8
    return {
        "tokens": T, "experts": E, "top_k": k, "H": H, "N": N,
        "padding_share": round(1 - T * k / used, 4),
        "grouped_tflops": round(flop / t_grp / 1e12, 1),
        "per_expert_launches_tflops": round(flop / t_loop / 1e12, 1),
        "dense_same_rows_tflops": round(flop / t_dense / 1e12, 1),
        "route_gbps": round(route_bytes / t_route / 1e9, 1),
        "permute_gbps": round(move_bytes / t_perm / 1e9, 1),
        "combine_gbps": round(comb_bytes / t_comb / 1e9, 1),
        "route_us": round(t_route * 1e6, 1), "permute_us": round(t_perm * 1e6, 1),
        "combine_us": round(t_comb * 1e6, 1),
    }


def steps(model, seq, n, warmup, layers=None):
    from distributed_training_guide_b200.engine import TrainEngine

    eng = TrainEngine.create(model, parallelism="single", batch_size=1, seq_length=seq, lr=1e-4, device="cuda",
                             num_layers=layers)
    try:
        batch = eng.synthetic_batch(seed=0)
        for _ in range(warmup):
            eng.step(batch)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        losses = [eng.step(batch) for _ in range(n)]
        b.record()
        b.synchronize()
        dt = a.elapsed_time(b) / 1e3 / n
        return {"model": model + (f"[layers={layers}]" if layers else ""), "seq": seq, "step_s": round(dt, 4),
                "tokens_per_s": round(seq / dt, 1),
                "peak_mem_gb": round(torch.cuda.max_memory_allocated() / 2**30, 2),
                "loss": float(losses[-1])}
    finally:
        eng.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seq", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--model", default="allenai/OLMoE-1B-7B-0924")
    ap.add_argument("--layers", type=int, default=None, help="train only the first N layers")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_olmoe.py measures on a GPU; none is visible")
    from distributed_training_guide_b200.models.configs import get_config

    cfg = get_config(a.model)
    rec = {"card": _card(), "kernels": kernels(a.seq, cfg.num_experts, cfg.num_experts_per_tok, cfg.hidden_size,
                                               2 * cfg.intermediate_size)}
    try:
        rec["train"] = steps(a.model, a.seq, a.steps, a.warmup, a.layers)
    except torch.OutOfMemoryError as e:
        rec["train"] = {"model": a.model, "error": f"out of memory: {str(e).splitlines()[0]}"}
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
