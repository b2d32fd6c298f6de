"""FP8 against bf16 for the Llama-2-7B decoder-layer projections on one H100.

    python bench_fp8.py [--tokens 4096] [--reps 20] [--rounds 5] [--steps 10] [--warmup 3] [--skip-e2e]

GEMM section: forward, dgrad and wgrad of the four projections (q|k|v, o, gate|up, down) at T tokens, timed with CUDA
events for the bf16 wgmma kernel, the fp8 wgmma kernel alone, the fp8 kernel together with the amax and cast-transpose
kernels that feed it, and ``torch._scaled_mm`` (cuBLASLt) on the same fp8 operands.  Every shape is warmed up, the
implementations alternate inside each round, and the median over rounds is reported.  TFLOP/s are 2*M*N*K over the
measured time; the cast kernels are reported in GB/s of the bytes they must move.

End-to-end section: ``TrainEngine`` on one GPU, Llama-2-7B, S 4096, B 1, run bf16, fp8, bf16, fp8, each in a process
of its own so that exactly one engine holds device memory (two 7B engines do not fit in 80 GB, and an engine's
symmetric-memory arena lives as long as its process); ms/step, tokens/s and peak memory of each run.

The card's name, power limit and SM clocks are read in the same run.  Prints one JSON record as the last line.
"""
from __future__ import annotations

import argparse
import json
import statistics
import subprocess
import sys
import time

import torch

from distributed_training_guide_b200 import _ext, ops

E4M3, E5M2 = torch.float8_e4m3fn, torch.float8_e5m2
HBM_GBPS = 3350.0  # H100 SXM data sheet

# Llama-2-7B: hidden 4096, intermediate 11008, 32 heads of 128 (no GQA)
PROJECTIONS = {"qkv": (12288, 4096), "o": (4096, 4096), "gate_up": (22016, 4096), "down": (4096, 11008)}


def gpu_info():
    q = ["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"]
    try:
        line = subprocess.run(q, capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, sm, sm_max = [s.strip() for s in line.split(",")]
        return {"name": name, "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max}
    except Exception as e:  # the numbers below still stand, but without their card
        return {"name": torch.cuda.get_device_name(), "error": repr(e)}


def time_ms(fn, reps):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(reps):
        fn()
    e.record()
    e.synchronize()
    return s.elapsed_time(e) / reps


def bench_alternating(impls, reps, rounds):
    """{name: median ms} over ``rounds`` rounds; inside a round every implementation runs ``reps`` times, in turn."""
    for fn in impls.values():   # warm-up: module load, tensor maps, cuBLASLt heuristics
        fn()
        fn()
    torch.cuda.synchronize()
    times = {k: [] for k in impls}
    for _ in range(rounds):
        for k, fn in impls.items():
            times[k].append(time_ms(fn, reps))
    return {k: statistics.median(v) for k, v in times.items()}


def gemm_section(T, reps, rounds):
    C = _ext.load(True)
    dev = torch.device("cuda")
    g = torch.Generator(device=dev).manual_seed(0)
    rows, passes = [], []
    for name, (N, K) in PROJECTIONS.items():
        x = torch.randn(T, K, device=dev, generator=g).to(torch.bfloat16)
        w = (0.02 * torch.randn(N, K, device=dev, generator=g)).to(torch.bfloat16)
        dy = (1e-3 * torch.randn(T, N, device=dev, generator=g)).to(torch.bfloat16)
        x8, x8t, sx = ops.fp8_cast(x, E4M3)
        w8, w8t, sw = ops.fp8_cast(w, E4M3)
        dy8, dy8t, sdy = ops.fp8_cast(dy, E5M2)
        y = torch.empty(T, N, dtype=torch.bfloat16, device=dev)
        dx = torch.empty(T, K, dtype=torch.bfloat16, device=dev)
        dw = torch.empty(N, K, dtype=torch.bfloat16, device=dev)

        def cast(t, fmt):
            return lambda: C.fp8_cast_transpose(t, C.fp8_amax(t), fmt == E5M2, True, True)

        casts = {"x": (x, E4M3), "w": (w, E4M3), "dy": (dy, E5M2)}
        cast_ms = bench_alternating({k: cast(t, f) for k, (t, f) in casts.items()}, reps, rounds)
        amax_ms = bench_alternating({k: (lambda t=t: C.fp8_amax(t)) for k, (t, _) in casts.items()}, reps, rounds)
        for k, (t, _) in casts.items():
            n = t.numel()
            rows.append({"projection": name, "kind": f"cast_{k}", "shape": list(t.shape),
                         "amax_ms": amax_ms[k], "amax_gbps": 2 * n / amax_ms[k] / 1e6,
                         "amax_cast_ms": cast_ms[k], "amax_cast_gbps": 6 * n / cast_ms[k] / 1e6,
                         "amax_cast_of_hbm_peak": 6 * n / cast_ms[k] / 1e6 / HBM_GBPS})
        gemms = {
            # pass: (M, N, K, bf16 call, fp8 call, _scaled_mm call, casts charged to the pass)
            "fwd": (T, N, K, lambda: C.gemm(x, w, y, False, True, False),
                    lambda: C.gemm_fp8(x8, w8, y, sx, sw, False),
                    lambda: torch._scaled_mm(x8, w8.t(), scale_a=sx, scale_b=sw, out_dtype=torch.bfloat16),
                    ("x", "w")),
            "dgrad": (T, K, N, lambda: C.gemm(dy, w, dx, False, False, False),
                      lambda: C.gemm_fp8(dy8, w8t, dx, sdy, sw, False),
                      lambda: torch._scaled_mm(dy8, w8t.t(), scale_a=sdy, scale_b=sw, out_dtype=torch.bfloat16),
                      ("dy",)),
            "wgrad": (N, K, T, lambda: C.gemm(dy, x, dw, True, False, False),
                      lambda: C.gemm_fp8(dy8t, x8t, dw, sdy, sx, False),
                      lambda: torch._scaled_mm(dy8t, x8t.t(), scale_a=sdy, scale_b=sx, out_dtype=torch.bfloat16),
                      ()),
        }
        for kind, (M, Nn, Kk, f_bf16, f_fp8, f_smm, charged) in gemms.items():
            ms = bench_alternating({"bf16": f_bf16, "fp8": f_fp8, "scaled_mm": f_smm}, reps, rounds)
            flop = 2.0 * M * Nn * Kk
            with_casts = ms["fp8"] + sum(cast_ms[c] for c in charged)
            rows.append({"projection": name, "kind": kind, "M": M, "N": Nn, "K": Kk,
                         "bf16_ms": ms["bf16"], "fp8_ms": ms["fp8"], "fp8_with_casts_ms": with_casts,
                         "scaled_mm_ms": ms["scaled_mm"],
                         "bf16_tflops": flop / ms["bf16"] / 1e9, "fp8_tflops": flop / ms["fp8"] / 1e9,
                         "fp8_with_casts_tflops": flop / with_casts / 1e9,
                         "scaled_mm_tflops": flop / ms["scaled_mm"] / 1e9,
                         "fp8_speedup": ms["bf16"] / ms["fp8"], "fp8_with_casts_speedup": ms["bf16"] / with_casts})
        del x, w, dy, x8, x8t, w8, w8t, dy8, dy8t, y, dx, dw
        torch.cuda.empty_cache()
    # one layer's projections, forward and backward
    tot = {k: 0.0 for k in ("bf16", "fp8", "fp8_with_casts", "scaled_mm")}
    for r in rows:
        if "bf16_ms" in r:
            for k in tot:
                tot[k] += r[f"{k}_ms"]
    passes.append({"layer_projections_ms": tot})
    return rows, passes


def e2e_run(fp8, steps, warmup, seq, batch):
    from distributed_training_guide_b200.engine import TrainEngine

    dev = torch.device("cuda", 0)
    eng = TrainEngine.create("meta-llama/Llama-2-7b-hf", parallelism="single", batch_size=batch, seq_length=seq,
                             device="cuda", fp8=fp8)
    batches = [eng.synthetic_batch(seed=i) for i in range(steps + warmup)]
    for b in batches[:warmup]:
        loss = eng.step(b)
    torch.cuda.synchronize(dev)
    t0 = time.perf_counter()
    for b in batches[warmup:]:
        loss = eng.step(b)
    torch.cuda.synchronize(dev)
    ms = (time.perf_counter() - t0) * 1e3 / steps
    free, total = torch.cuda.mem_get_info(dev)
    out = {"fp8": fp8, "ms_per_step": ms, "tokens_per_s": batch * seq / ms * 1e3, "loss": float(loss),
           "peak_alloc_gb": torch.cuda.max_memory_allocated(dev) / 1e9,
           "peak_reserved_gb": torch.cuda.max_memory_reserved(dev) / 1e9,
           "device_used_gb": (total - free) / 1e9}
    eng.close()
    return out


def e2e_in_subprocess(fp8, a):
    cmd = [sys.executable, __file__, "--e2e-one", "fp8" if fp8 else "bf16", "--steps", str(a.steps), "--warmup",
           str(a.warmup), "--seq-length", str(a.seq_length), "--batch-size", str(a.batch_size)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        return {"fp8": fp8, "error": (r.stdout + r.stderr).strip().splitlines()[-1]}
    return json.loads(r.stdout.strip().splitlines()[-1])


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--tokens", type=int, default=4096)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--seq-length", type=int, default=4096)
    ap.add_argument("--batch-size", type=int, default=1)
    ap.add_argument("--skip-e2e", action="store_true")
    ap.add_argument("--e2e-one", choices=("bf16", "fp8"), help=argparse.SUPPRESS)   # one end-to-end run, then exit
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_fp8.py measures on a CUDA device; none is visible")
    if a.e2e_one:
        print(json.dumps(e2e_run(a.e2e_one == "fp8", a.steps, a.warmup, a.seq_length, a.batch_size)))
        return
    info = gpu_info()
    print(f"# {info}", flush=True)
    rows, passes = gemm_section(a.tokens, a.reps, a.rounds)
    for r in rows:
        print("# " + json.dumps(r), flush=True)
    e2e = []
    if not a.skip_e2e:
        for fp8 in (False, True, False, True):
            r = e2e_in_subprocess(fp8, a)
            print("# " + json.dumps(r), flush=True)
            e2e.append(r)
    summary = {}
    fwd = [r for r in rows if r.get("kind") == "fwd"]
    summary["fwd_fp8_speedup_min"] = min(r["fp8_speedup"] for r in fwd)
    if e2e:
        for key in ("ms_per_step", "tokens_per_s", "device_used_gb", "peak_alloc_gb"):
            for fp8 in (False, True):
                vals = [r[key] for r in e2e if r["fp8"] == fp8 and key in r]
                if vals:
                    summary[f"{'fp8' if fp8 else 'bf16'}_{key}"] = statistics.mean(vals)
    print(json.dumps({"gpu": info, "tokens": a.tokens, "gemm": rows, "layer": passes, "e2e": e2e,
                      "summary": summary}))


if __name__ == "__main__":
    main()
