"""The q|k|v bias on one H100: the GEMM's bias epilogue, the bias-gradient kernel, and Qwen2.5 training steps.

    python bench_qwen2.py [--reps 20] [--rounds 5] [--steps 5] [--warmup 2] [--layers N] [--skip-e2e]

GEMM section: the q|k|v projection at Qwen2.5-7B (T 4096, K 3584, N 4608) and Qwen2.5-0.5B (T 4096, K 896, N 1152)
shapes, timed as
  * ``no_bias``: the plain wgmma GEMM (what a Llama layer runs);
  * ``bias_epilogue``: the same GEMM adding the bias before its one rounding;
  * ``gemm_then_add``: the plain GEMM, then ATen's broadcast ``add_`` of the bias (a second pass over T x N);
  * ``prefilled_accumulate``: C filled with the broadcast bias, then the GEMM in accumulate mode (the kernel loads C).
TFLOP/s counts 2 T K N over the median time of the case.

Bias-gradient section: ``bias_grad`` (per-CTA fp32 partial rows + the fixed-order column sum) against ATen's
``dy.float().sum(0)`` at the same two shapes, in GB/s of the T x N bf16 read.

CUDA-event medians over rounds, the cases alternating inside each round.  End-to-end section: device-timed tokens/s
and peak memory of single-GPU ``TrainEngine`` steps of Qwen/Qwen2.5-0.5B and -7B at S 4096, B 1, each in a process of
its own; when the whole 7B model does not fit, it runs again with ``--layers`` of its 28 decoder layers and the record
says so.  The card's name and power limit are read in the same run.  Prints one JSON record as the last line.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_window import gpu_info  # noqa: E402

SHAPES = {"Qwen2.5-7B": (4096, 3584, 4608), "Qwen2.5-0.5B": (4096, 896, 1152)}   # T, K, N of the q|k|v GEMM
S = 4096


def _time_ms(fn, n):
    import torch

    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(n):
        fn()
    e.record()
    e.synchronize()
    return s.elapsed_time(e) / n


def _medians(cases, reps, rounds):
    for fn in cases.values():
        _time_ms(fn, 3)
    times = {k: [] for k in cases}
    for _ in range(rounds):
        for k, fn in cases.items():
            times[k].append(_time_ms(fn, reps))
    return times


def gemm_section(reps, rounds):
    import torch

    from distributed_training_guide_b200 import _ext

    C = _ext.load(required=True)
    out = []
    for name, (T, K, N) in SHAPES.items():
        g = torch.Generator(device="cuda").manual_seed(0)
        x = torch.randn(T, K, device="cuda", generator=g).to(torch.bfloat16)
        w = (torch.randn(N, K, device="cuda", generator=g) * 0.02).to(torch.bfloat16)
        b = torch.randn(N, device="cuda", generator=g).to(torch.bfloat16)
        y = torch.empty(T, N, device="cuda", dtype=torch.bfloat16)

        def prefilled():
            y.copy_(b.expand(T, N))
            C.gemm(x, w, y, False, True, True, 0)

        def then_add():
            C.gemm(x, w, y, False, True, False, 0)
            y.add_(b)

        cases = {
            "no_bias": lambda: C.gemm(x, w, y, False, True, False, 0),
            "bias_epilogue": lambda: C.gemm(x, w, y, False, True, False, 0, bias=b),
            "gemm_then_add": then_add,
            "prefilled_accumulate": prefilled,
        }
        times = _medians(cases, reps, rounds)
        flops = 2.0 * T * K * N
        for k in cases:
            med = statistics.median(times[k])
            rec = {"shape": name, "T": T, "K": K, "N": N, "case": k, "ms_median": round(med, 4),
                   "ms_min": round(min(times[k]), 4), "ms_max": round(max(times[k]), 4),
                   "TFLOP_per_s": round(flops / (med * 1e-3) / 1e12, 1)}
            out.append(rec)
            print(f"{name:13s} {k:22s} {med * 1e3:9.1f} us  {rec['TFLOP_per_s']:6.1f} TFLOP/s", flush=True)
    return out


def bias_grad_section(reps, rounds):
    import torch

    from distributed_training_guide_b200 import _ext

    C = _ext.load(required=True)
    out = []
    for name, (T, _, N) in SHAPES.items():
        dy = torch.randn(T, N, device="cuda").to(torch.bfloat16)
        cases = {"bias_grad": lambda: C.bias_grad(dy), "aten_float_sum": lambda: dy.float().sum(0)}
        times = _medians(cases, reps, rounds)
        nbytes = T * N * 2
        for k in cases:
            med = statistics.median(times[k])
            gbs = nbytes / (med * 1e-3) / 1e9
            rec = {"shape": name, "T": T, "N": N, "case": k, "bytes": nbytes, "ms_median": round(med, 4),
                   "ms_min": round(min(times[k]), 4), "ms_max": round(max(times[k]), 4), "GB_per_s": round(gbs, 1)}
            out.append(rec)
            print(f"{name:13s} {k:22s} {med * 1e3:9.1f} us  {gbs:7.1f} GB/s", flush=True)
    return out


def e2e_run(model, layers, steps, warmup):
    import torch

    from distributed_training_guide_b200.engine import TrainEngine

    dev = torch.device("cuda", 0)
    kw = {"num_layers": layers} if layers else {}
    eng = TrainEngine.create(model, parallelism="single", batch_size=1, seq_length=S, device="cuda", **kw)
    batches = [eng.synthetic_batch(seed=i) for i in range(steps + warmup)]
    for b in batches[:warmup]:
        loss = eng.step(b)
    torch.cuda.synchronize(dev)
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0 = time.perf_counter()
    s.record()
    for b in batches[warmup:]:
        loss = eng.step(b)
    e.record()
    torch.cuda.synchronize(dev)
    host_ms = (time.perf_counter() - t0) * 1e3 / steps
    dev_ms = s.elapsed_time(e) / steps
    out = {"model": model, "num_layers": layers or eng.config.num_hidden_layers, "S": S, "B": 1,
           "ms_per_step_device": round(dev_ms, 2), "ms_per_step_host": round(host_ms, 2),
           "tokens_per_s_device": round(S / dev_ms * 1e3), "loss": float(loss),
           "peak_alloc_gb": round(torch.cuda.max_memory_allocated(dev) / 1e9, 2)}
    eng.close()
    return out


def e2e_in_subprocess(model, layers, a):
    cmd = [sys.executable, __file__, "--e2e-one", model, "--steps", str(a.steps), "--warmup", str(a.warmup),
           "--layers", str(layers)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write((r.stdout + r.stderr)[-2000:])
        return {"model": model, "num_layers": layers or "all", "error": (r.stdout + r.stderr).strip().splitlines()[-1]}
    return json.loads(r.stdout.strip().splitlines()[-1])


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--layers", type=int, default=0, help="decoder layers of the 7B step when all 28 do not fit")
    ap.add_argument("--skip-e2e", action="store_true")
    ap.add_argument("--e2e-one", default=None, help=argparse.SUPPRESS)   # one end-to-end run of this model, then exit
    a = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        sys.exit("bench_qwen2.py measures on a CUDA device; none is visible")
    from distributed_training_guide_b200 import _ext

    _ext.load(required=True)
    if a.e2e_one:
        print(json.dumps(e2e_run(a.e2e_one, a.layers, a.steps, a.warmup)))
        return
    info = gpu_info()
    print(f"gpu: {info}", flush=True)
    gemms = gemm_section(a.reps, a.rounds)
    grads = bias_grad_section(a.reps, a.rounds)
    e2e = "not measured"
    if not a.skip_e2e:
        e2e = []
        for model in ("Qwen/Qwen2.5-0.5B", "Qwen/Qwen2.5-7B"):
            e2e.append(e2e_in_subprocess(model, 0, a))
            print(f"e2e: {e2e[-1]}", flush=True)
            if "error" in e2e[-1]:
                e2e[-1]["fits_in_80GB"] = False
                e2e.append(e2e_in_subprocess(model, a.layers or 14, a))
                print(f"e2e (reduced to {a.layers or 14} layers): {e2e[-1]}", flush=True)
    print(json.dumps({"gpu": info, "gemm": gemms, "bias_grad": grads, "e2e": e2e}))


if __name__ == "__main__":
    main()
