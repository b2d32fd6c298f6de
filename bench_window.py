"""Sliding-window attention on one H100: Mistral-7B attention shapes and a Mistral-7B training step, window against
causal.

    python bench_window.py [--reps 5] [--rounds 3] [--steps 5] [--warmup 2] [--e2e-layers 16] [--skip-e2e]

Kernel section: B 1, 32 q heads : 8 kv heads, head_dim 128 (Mistral-7B), S 4096, 8192, 16384 and 32768.  For each S
it times the forward alone (``ops.attention_qkv`` under ``no_grad``) and forward + backward (``torch.autograd.grad``
through it) with CUDA events, for causal attention and for a window of 4096.  Cases alternate inside each round, and
the median over rounds is reported with TFLOP/s over the *visible* (q, k) pairs: causal attention has S(S+1)/2 of
them, a window of W has sum_q min(q + 1, W).  At S 4096 a window of 4096 covers the sequence and runs the causal
kernels, so the two rows there time the same code.

End-to-end section: one Mistral-7B single-GPU ``TrainEngine`` step (S 8192, B 1) with the window and with it removed,
each in a process of its own, alternating.  32 layers with their AdamW state and S 8192 activations need more than an
80 GB card, so the model keeps ``--e2e-layers`` of its 32 layers (16 by default; the record says how many).  The
card's name and power limit are read in the same run.  Prints one JSON record as the last line.
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

NH, NKV, D, WINDOW = 32, 8, 128, 4096
MODEL = "mistralai/Mistral-7B-v0.1"


def gpu_info():
    q = ["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"]
    try:
        line = subprocess.run(q, capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, sm, sm_max = [s.strip() for s in line.split(",")]
        return {"name": name, "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max}
    except Exception as e:  # the numbers still stand, but without their card
        return {"error": repr(e)}


def visible_pairs(S, window):
    """(q, k) pairs with max(0, q - W + 1) <= k <= q."""
    if window is None or window >= S:
        return S * (S + 1) // 2
    return window * (window + 1) // 2 + (S - window) * window


def flop(S, window, backward):
    """Matmul FLOPs over the visible pairs: QK^T and PV forward, plus QK^T again, dP, dV, dQ and dK backward."""
    return (7 if backward else 2) * 2 * D * NH * visible_pairs(S, window)


def kernel_section(reps, rounds):
    import torch

    from distributed_training_guide_b200 import ops

    out = []
    for S in (4096, 8192, 16384, 32768):
        g = torch.Generator(device="cuda").manual_seed(0)
        qkv = torch.randn(1, S, NH + 2 * NKV, D, device="cuda", generator=g).to(torch.bfloat16).requires_grad_(True)
        do = torch.randn(1, S, NH, D, device="cuda", generator=g).to(torch.bfloat16)
        cases = [(w, bwd) for bwd in (False, True) for w in (None, WINDOW)]

        def run(window, bwd):
            if bwd:
                o = ops.attention_qkv(qkv, NH, NKV, window=window)
                return torch.autograd.grad(o, qkv, do)
            with torch.no_grad():
                return ops.attention_qkv(qkv, NH, NKV, window=window)

        def time_ms(case, n):
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            for _ in range(n):
                run(*case)
            e.record()
            e.synchronize()
            return s.elapsed_time(e) / n

        for c in cases:
            time_ms(c, 2)
        times = {c: [] for c in cases}
        for _ in range(rounds):
            for c in cases:
                times[c].append(time_ms(c, reps))
        for c in cases:
            window, bwd = c
            med = statistics.median(times[c])
            causal = statistics.median(times[(None, bwd)])
            rec = {"S": S, "nh": NH, "nkv": NKV, "window": window, "pass": "fwd+bwd" if bwd else "fwd",
                   "visible_pairs_per_head": visible_pairs(S, window), "ms_median": round(med, 4),
                   "ms_min": round(min(times[c]), 4), "ms_max": round(max(times[c]), 4),
                   "tflops_visible": round(flop(S, window, bwd) / med / 1e9, 1),
                   "speedup_vs_causal": round(causal / med, 3)}
            out.append(rec)
            print(f"S {S:5d} {rec['pass']:7s} window {str(window):5s} {med:9.3f} ms  {rec['tflops_visible']:6.1f} "
                  f"TFLOP/s  x{rec['speedup_vs_causal']:.2f}", flush=True)
        del qkv, do
        torch.cuda.empty_cache()
    return out


def e2e_run(window_on, layers, steps, warmup):
    import torch

    from distributed_training_guide_b200.engine import TrainEngine

    S = 8192
    dev = torch.device("cuda", 0)
    eng = TrainEngine.create(MODEL, parallelism="single", batch_size=1, seq_length=S, device="cuda",
                             num_layers=layers)
    if not window_on:
        for layer in eng.model.model.layers:
            layer.self_attn.sliding_window = None
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
    ms = (time.perf_counter() - t0) * 1e3 / steps
    out = {"window": WINDOW if window_on else None, "num_layers": layers, "S": S, "ms_per_step": round(ms, 2),
           "ms_per_step_device": round(s.elapsed_time(e) / steps, 2), "tokens_per_s": round(S / ms * 1e3),
           "loss": float(loss), "peak_alloc_gb": round(torch.cuda.max_memory_allocated(dev) / 1e9, 2),
           "peak_reserved_gb": round(torch.cuda.max_memory_reserved(dev) / 1e9, 2)}
    eng.close()
    return out


def e2e_in_subprocess(window_on, a):
    cmd = [sys.executable, __file__, "--e2e-one", "on" if window_on else "off", "--steps", str(a.steps),
           "--warmup", str(a.warmup), "--e2e-layers", str(a.e2e_layers)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        return {"window": WINDOW if window_on else None, "num_layers": a.e2e_layers,
                "error": (r.stdout + r.stderr).strip().splitlines()[-1]}
    return json.loads(r.stdout.strip().splitlines()[-1])


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--e2e-layers", type=int, default=16)
    ap.add_argument("--skip-e2e", action="store_true")
    ap.add_argument("--e2e-one", choices=("off", "on"), help=argparse.SUPPRESS)   # one end-to-end run, then exit
    a = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        sys.exit("bench_window.py measures on a CUDA device; none is visible")
    from distributed_training_guide_b200 import _ext

    _ext.load(required=True)
    if a.e2e_one:
        print(json.dumps(e2e_run(a.e2e_one == "on", a.e2e_layers, a.steps, a.warmup)))
        return
    info = gpu_info()
    print(f"gpu: {info}", flush=True)
    kernels = kernel_section(a.reps, a.rounds)
    if a.skip_e2e:
        e2e = "not measured"
    else:
        e2e = []
        for on in (False, True, False, True):
            e2e.append(e2e_in_subprocess(on, a))
            print(f"e2e: {e2e[-1]}", flush=True)
    summary = {}
    for r in kernels:
        if r["window"] is not None:
            summary[f"S{r['S']}_{r['pass']}_speedup_vs_causal"] = r["speedup_vs_causal"]
    for on in (False, True):
        vals = [r["ms_per_step"] for r in (e2e if isinstance(e2e, list) else []) if "ms_per_step" in r
                and (r["window"] is not None) == on]
        summary[f"e2e_ms_per_step_{'window' if on else 'causal'}"] = round(statistics.mean(vals), 2) if vals \
            else "not measured"
    print(json.dumps({"gpu": info, "kernels": kernels, "e2e": e2e, "summary": summary}))


if __name__ == "__main__":
    main()
