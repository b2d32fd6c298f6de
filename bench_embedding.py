"""Embedding backward on one H100: the time of the default (non-deterministic) backward, as the model runs it.

    python bench_embedding.py [--root DIR] [--reps 50] [--rounds 5]

Times ``torch.autograd.grad`` through ``ops.embedding`` (the gather's graph is built once, so only the backward runs:
allocation of the gradient, the kernels, and autograd's own work) with CUDA events, for B 1 and 4 at S 4096, H 4096,
V 32000 and three id distributions: uniform, Zipf(1.0) (the shape of real text) and pad-heavy (half the tokens one
id).  Every case is warmed up, the cases alternate inside each round, and the median over rounds is reported, with the
bytes the backward must move (read dout, write the table) over that time.

A second section times the hidden-parallel (tensor-parallel) backward, ``tp_embed_bwd``, with its ranks emulated on
this one GPU: T 8192, H 4096, V 128256 and N 2, 4 and 8 ranks, Zipf(1.0) ids.  Every rank's [T / N, H] gradient buffer
and [V, H / N] table shard is a separate tensor here, and the N ranks' calls run back to back; the time reported is per
rank (the N calls over N), in overwrite mode as the first write of a step runs it.  The pulls read local memory, so the
NVLink traffic of a real multi-GPU run is not measured.

``--root DIR`` imports the package from another checkout (with its extension built), so two versions can be timed
by alternating runs of this script.  The card's name and power limit are read in the same run.  Prints one JSON record
as the last line.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys


def gpu_info():
    q = ["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"]
    try:
        line = subprocess.run(q, capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, sm, sm_max = [s.strip() for s in line.split(",")]
        return {"name": name, "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max}
    except Exception as e:  # the numbers still stand, but without their card
        return {"error": repr(e)}


def make_ids(kind, T, V, g):
    import torch

    if kind == "zipf":
        p = torch.arange(1, V + 1, device="cuda", dtype=torch.float32).pow(-1.0)
        return torch.randperm(V, device="cuda", generator=g)[torch.multinomial(p, T, replacement=True, generator=g)]
    ids = torch.randint(0, V, (T,), device="cuda", generator=g)
    if kind == "pad":
        ids[torch.randperm(T, device="cuda", generator=g)[:T // 2]] = 0
    return ids


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--root", default=os.path.dirname(os.path.abspath(__file__)))
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=5)
    a = ap.parse_args()
    sys.path.insert(0, os.path.abspath(a.root))
    import torch

    from distributed_training_guide_b200 import _ext, ops

    assert torch.cuda.is_available(), "bench_embedding.py needs a CUDA device"
    _ext.load(required=True)
    V, H, S = 32000, 4096, 4096
    g = torch.Generator(device="cuda").manual_seed(0)
    w = (0.02 * torch.randn(V, H, device="cuda", generator=g)).to(torch.bfloat16).requires_grad_(True)
    cases = {}
    for B in (1, 4):
        dout = (1e-3 * torch.randn(B, S, H, device="cuda", generator=g)).to(torch.bfloat16)
        for kind in ("uniform", "zipf", "pad"):
            ids = make_ids(kind, B * S, V, g).view(B, S)
            out = ops.embedding(ids, w)
            cases[f"B{B}-{kind}"] = (out, dout)

    def run(case):
        out, dout = cases[case]
        return torch.autograd.grad(out, w, dout, retain_graph=True)

    def time_ms(case, reps):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(reps):
            run(case)
        e.record()
        e.synchronize()
        return s.elapsed_time(e) / reps

    for c in cases:
        time_ms(c, 3)
    times = {c: [] for c in cases}
    for _ in range(a.rounds):
        for c in cases:
            times[c].append(time_ms(c, a.reps))
    res = {}
    for c, t in times.items():
        T = cases[c][1].shape[0] * S
        med = statistics.median(t)
        moved = T * H * 2 + V * H * 2       # read dout, write every row of the table
        res[c] = {"ms_median": round(med, 4), "ms_min": round(min(t), 4), "ms_max": round(max(t), 4),
                  "GB_per_s_min_traffic": round(moved / med / 1e6, 1)}
        print(f"{c:12s} {med:8.4f} ms  (min {min(t):.4f}, max {max(t):.4f})  {res[c]['GB_per_s_min_traffic']} GB/s")
    del cases, w
    tp = tp_section(a, g)
    print(json.dumps({"root": os.path.abspath(a.root), "gpu": gpu_info(), "V": V, "H": H, "S": S, "cases": res,
                      "tp": tp}))


def tp_section(a, g):
    import torch

    from distributed_training_guide_b200 import _ext

    C = _ext.load(required=True)
    V, H, T = 128256, 4096, 8192
    ids = make_ids("zipf", T, V, g)
    dx = (1e-3 * torch.randn(T, H, device="cuda", generator=g)).to(torch.bfloat16)
    res = {}
    for N in (2, 4, 8):
        rpp, Hl = T // N, H // N
        parts = [dx[k * rpp:(k + 1) * rpp].clone() for k in range(N)]
        ptrs = [p.data_ptr() for p in parts]
        dws = [torch.empty(V, Hl, device="cuda", dtype=torch.bfloat16) for _ in range(N)]

        def run():
            for k in range(N):
                try:
                    C.tp_embed_bwd(ids, ptrs, dws[k], rpp, H, k, False)
                except TypeError:    # a checkout whose binding takes no mode: the caller zeroed the shard
                    dws[k].zero_()
                    C.tp_embed_bwd(ids, ptrs, dws[k], rpp, H, k)

        def time_ms(reps):
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            for _ in range(reps):
                run()
            e.record()
            e.synchronize()
            return s.elapsed_time(e) / reps / N

        time_ms(3)
        t = [time_ms(max(a.reps // 5, 2)) for _ in range(a.rounds)]
        med = statistics.median(t)
        res[f"N{N}"] = {"ms_per_rank_median": round(med, 4), "ms_min": round(min(t), 4), "ms_max": round(max(t), 4)}
        print(f"tp N{N:<2d}       {med:8.4f} ms per rank  (min {min(t):.4f}, max {max(t):.4f})")
        del parts, dws
    return {"V": V, "H": H, "T": T, "ids": "zipf1.0", "cases": res}


if __name__ == "__main__":
    main()
