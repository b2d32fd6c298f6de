"""The bf16 wgmma GEMM at the shapes of one Llama-2-7B training step (T = 4096 tokens) against cuBLAS.

    python bench_gemm.py [--tokens 4096] [--reps 10] [--rounds 7]
    python bench_gemm.py --baseline DIR [--pairs 3]     # + another build of the package, for before / after

Shapes: q|k|v, o, gate|up, down and the lm_head, each as the forward ``nt`` (Y = X . W^T), the dgrad ``nn``
(dX = dY . W) and the wgrad ``tn`` (dW = dY^T . X), called the way ``ops`` calls them; the wgrads also in accumulate
mode (dW += ..., every micro-batch after the first of gradient accumulation).  cuBLAS is ``torch.matmul`` (``addmm_``
for accumulate) on the same operands and layouts.  Every shape is warmed up, the two implementations alternate inside
each round, and the median over rounds is reported as TFLOP/s (2 M N K over the time).

Fixed cost per tile: on a 4096 x 4096 output, ``t(K) = a + b K`` is fitted at K = 2048, 4096, 8192 (forward layout,
both modes).  ``b`` is the mainloop's time per unit of K, ``a`` what a GEMM costs whatever its K; divided by the tile
waves (tiles over co-resident CTAs) ``a`` is the fixed cost of one tile: launch, pipeline fill and the epilogue.

``--baseline DIR``: DIR is another checkout of this repository with its extension built (``bench_fp8.py`` and
``distributed_training_guide_b200/_C.so`` are read from it).  Each measurement then runs in a process of its own,
alternating this tree and DIR ``--pairs`` times (two builds of the extension cannot share a process), and the medians
over the pairs are reported side by side.

The card's name, power limit and SM clocks are read in the same run.  Prints one JSON record as the last line.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))

# Llama-2-7B: hidden 4096, intermediate 11008, vocabulary 32000, 32 heads of 128 (no GQA); (N, K) of each weight
WEIGHTS = {"qkv": (12288, 4096), "o": (4096, 4096), "gate_up": (22016, 4096), "down": (4096, 11008),
           "lm_head": (32000, 4096)}
FIT_K = (2048, 4096, 8192)
FIT_MN = 4096


def measure(root, tokens, reps, rounds):
    """One process, one build: {case: {"M", "N", "K", "ours_ms", "cublas_ms"}} plus the card's state."""
    sys.path.insert(0, root)
    import torch

    from bench_fp8 import bench_alternating, gpu_info
    from distributed_training_guide_b200 import _ext

    C = _ext.load(True)
    torch.backends.cuda.matmul.allow_bf16_reduced_precision_reduction = False
    dev = torch.device("cuda")
    g = torch.Generator(device=dev).manual_seed(0)
    T = tokens
    rows = {}

    def run(case, M, N, K, ours, cublas):
        ms = bench_alternating({"ours": ours, "cublas": cublas}, reps, rounds)
        rows[case] = {"M": M, "N": N, "K": K, "ours_ms": ms["ours"], "cublas_ms": ms["cublas"]}

    for name, (N, K) in WEIGHTS.items():
        x = torch.randn(T, K, device=dev, generator=g).to(torch.bfloat16)
        w = (0.02 * torch.randn(N, K, device=dev, generator=g)).to(torch.bfloat16)
        dy = (1e-3 * torch.randn(T, N, device=dev, generator=g)).to(torch.bfloat16)
        y = torch.empty(T, N, dtype=torch.bfloat16, device=dev)
        dx = torch.empty(T, K, dtype=torch.bfloat16, device=dev)
        dw = torch.zeros(N, K, dtype=torch.bfloat16, device=dev)
        run(f"{name}/fwd", T, N, K, lambda: C.gemm(x, w, y, False, True, False), lambda: torch.matmul(x, w.t(), out=y))
        run(f"{name}/dgrad", T, K, N, lambda: C.gemm(dy, w, dx, False, False, False), lambda: torch.matmul(dy, w, out=dx))
        run(f"{name}/wgrad", N, K, T, lambda: C.gemm(dy, x, dw, True, False, False),
            lambda: torch.matmul(dy.t(), x, out=dw))
        run(f"{name}/wgrad_acc", N, K, T, lambda: C.gemm(dy, x, dw, True, False, True), lambda: dw.addmm_(dy.t(), x))
        del x, w, dy, y, dx, dw
        torch.cuda.empty_cache()
    for K in FIT_K:
        a = torch.randn(FIT_MN, K, device=dev, generator=g).to(torch.bfloat16)
        b = torch.randn(FIT_MN, K, device=dev, generator=g).to(torch.bfloat16)
        c = torch.zeros(FIT_MN, FIT_MN, dtype=torch.bfloat16, device=dev)
        run(f"fit/K{K}", FIT_MN, FIT_MN, K, lambda: C.gemm(a, b, c, False, True, False),
            lambda: torch.matmul(a, b.t(), out=c))
        run(f"fit_acc/K{K}", FIT_MN, FIT_MN, K, lambda: C.gemm(a, b, c, False, True, True), lambda: c.addmm_(a, b.t()))
        del a, b, c
    return {"gpu": gpu_info(), "rows": rows, "sms": torch.cuda.get_device_properties(dev).multi_processor_count}


def fit(rows, prefix, key, sms):
    """Least-squares t(K) = a + b K over the fit shapes; a per tile wave of the 2-CTA (256 x 256 tile) kernel."""
    ks = [float(k) for k in FIT_K]
    ts = [rows[f"{prefix}/K{k}"][key] for k in FIT_K]
    km, tm = statistics.mean(ks), statistics.mean(ts)
    b = sum((k - km) * (t - tm) for k, t in zip(ks, ts)) / sum((k - km) ** 2 for k in ks)
    a = tm - b * km
    waves = -(-(FIT_MN // 256) ** 2 // (sms // 2))
    return {"intercept_ms": a, "slope_ms_per_k": b, "tile_waves": waves, "intercept_us_per_wave": 1e3 * a / waves}


def in_subprocess(root, a):
    cmd = [sys.executable, os.path.abspath(__file__), "--one", root, "--tokens", str(a.tokens), "--reps", str(a.reps),
           "--rounds", str(a.rounds)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        raise SystemExit(f"bench_gemm.py: the run on {root} failed")
    return json.loads(r.stdout.strip().splitlines()[-1])


def tflops(r, ms):
    return 2.0 * r["M"] * r["N"] * r["K"] / ms / 1e9


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--tokens", type=int, default=4096)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--baseline", metavar="DIR", default=None, help="another build of the package to compare with")
    ap.add_argument("--pairs", type=int, default=3)
    ap.add_argument("--one", metavar="ROOT", default=None, help=argparse.SUPPRESS)   # one measurement, then exit
    a = ap.parse_args()
    if a.one:
        print(json.dumps(measure(a.one, a.tokens, a.reps, a.rounds)))
        return
    import torch

    if not torch.cuda.is_available():
        sys.exit("bench_gemm.py measures on a CUDA device; none is visible")
    builds = {"this": ROOT}
    if a.baseline:
        builds["baseline"] = os.path.abspath(a.baseline)
    runs = {k: [] for k in builds}
    for _ in range(a.pairs if a.baseline else 1):
        for k, root in builds.items():
            runs[k].append(in_subprocess(root, a))
            print(f"# {k}: {json.dumps(runs[k][-1]['gpu'])}", flush=True)
    sms = runs["this"][0]["sms"]
    cases = list(runs["this"][0]["rows"])
    table = []
    for case in cases:
        r0 = runs["this"][0]["rows"][case]
        row = {"case": case, "M": r0["M"], "N": r0["N"], "K": r0["K"]}
        for k in builds:
            ours = [run["rows"][case]["ours_ms"] for run in runs[k]]
            row[f"{k}_ms"] = statistics.median(ours)
            row[f"{k}_spread_ms"] = max(ours) - min(ours)
            row[f"{k}_tflops"] = tflops(r0, row[f"{k}_ms"])
        cub = [run["rows"][case]["cublas_ms"] for k in builds for run in runs[k]]
        row["cublas_ms"] = statistics.median(cub)
        row["cublas_tflops"] = tflops(r0, row["cublas_ms"])
        if a.baseline:
            row["speedup"] = row["baseline_ms"] / row["this_ms"]
        table.append(row)
    fits = {}
    for k in builds:
        med = {case: {"t": statistics.median(run["rows"][case]["ours_ms"] for run in runs[k])} for case in cases}
        fits[k] = {p: fit(med, p, "t", sms) for p in ("fit", "fit_acc")}
    cub_med = {case: {"t": next(r["cublas_ms"] for r in table if r["case"] == case)} for case in cases}
    fits["cublas"] = {p: fit(cub_med, p, "t", sms) for p in ("fit", "fit_acc")}
    hdr = f"{'case':22s} {'M':>6s} {'N':>6s} {'K':>6s}" + "".join(f" {k + ' TF/s':>14s}" for k in builds)
    print("# " + hdr + f" {'cuBLAS TF/s':>12s}" + (" speedup" if a.baseline else ""))
    for r in table:
        line = f"{r['case']:22s} {r['M']:6d} {r['N']:6d} {r['K']:6d}"
        line += "".join(f" {r[f'{k}_tflops']:14.1f}" for k in builds) + f" {r['cublas_tflops']:12.1f}"
        if a.baseline:
            line += f" {r['speedup']:7.3f}"
        print("# " + line)
    for k, f in fits.items():
        print(f"# fixed cost {k}: " + json.dumps(f))
    print(json.dumps({"gpu": runs["this"][0]["gpu"], "tokens": a.tokens, "table": table, "fit": fits,
                      "pairs": a.pairs if a.baseline else 1}))


if __name__ == "__main__":
    main()
