"""Document-masked attention on one H100: forward + backward time against the number of documents in a row.

    python bench_docmask.py [--reps 10] [--rounds 5] [--steps 5] [--warmup 2] [--skip-e2e]

Times ``torch.autograd.grad`` through ``ops.attention_qkv`` (forward and backward, B 1) with CUDA events at S 4096 and
8192 for two geometries, Llama-2-7B (32 q heads : 32 kv heads) and Llama-3-8B (32 : 8), with these layouts of a row:
one document through the plain causal kernels, one document through the document-masking kernels, documents of
2048, 512 and 128 tokens, and a mixed layout (lengths drawn uniformly from 32..2048, seed 0, the last one cut at the
row's end).  Every case is warmed up, the cases of one shape alternate inside each round, and the median over rounds
is reported with the useful TFLOP/s (the causal FLOPs of each document, summed, over the time) and the speed-up over
one document through the plain kernels.

End-to-end section: one Llama-2-7B single-GPU training step (``TrainEngine``, S 4096, B 1) with and without
``document_masking`` on 512-token documents, each in a process of its own.  The card's name and power limit are read
in the same run.  Prints one JSON record as the last line.
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

GEOMETRIES = {"llama2-7b": (32, 32), "llama3-8b": (32, 8)}
D = 128


def gpu_info():
    q = ["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"]
    try:
        line = subprocess.run(q, capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, sm, sm_max = [s.strip() for s in line.split(",")]
        return {"name": name, "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max}
    except Exception as e:  # the numbers still stand, but without their card
        return {"error": repr(e)}


def layout_lengths(layout, S):
    """Document lengths of one row."""
    import random

    if layout in ("one-plain", "one-doc"):
        return [S]
    if layout.startswith("docs"):
        n = int(layout[4:])
        return [n] * (S // n)
    rng, out = random.Random(0), []
    while sum(out) < S:
        out.append(min(rng.randint(32, 2048), S - sum(out)))
    return out


def positions(lengths):
    import torch

    return torch.cat([torch.arange(n) for n in lengths])[None]


def useful_flop(lengths, nh):
    """Forward (QK^T, PV) + backward (QK^T again, dP, dV, dQ, dK) matmul FLOPs of causal attention per document."""
    pairs = sum(n * (n + 1) // 2 for n in lengths)
    return 7 * 2 * D * nh * pairs


def kernel_section(reps, rounds):
    import torch

    from distributed_training_guide_b200 import ops

    layouts = ["one-plain", "one-doc", "docs2048", "docs512", "docs128", "mixed"]
    out = []
    for geo, (nh, nkv) in GEOMETRIES.items():
        for S in (4096, 8192):
            g = torch.Generator(device="cuda").manual_seed(0)
            qkv = torch.randn(1, S, nh + 2 * nkv, D, device="cuda", generator=g).to(torch.bfloat16).requires_grad_(True)
            do = torch.randn(1, S, nh, D, device="cuda", generator=g).to(torch.bfloat16)
            ds = {lay: (None if lay == "one-plain" else ops.document_starts(positions(layout_lengths(lay, S)).cuda()))
                  for lay in layouts}

            def run(lay):
                o = ops.attention_qkv(qkv, nh, nkv, doc_start=ds[lay])
                return torch.autograd.grad(o, qkv, do)

            def time_ms(lay, n):
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record()
                for _ in range(n):
                    run(lay)
                e.record()
                e.synchronize()
                return s.elapsed_time(e) / n

            for lay in layouts:
                time_ms(lay, 2)
            times = {lay: [] for lay in layouts}
            for _ in range(rounds):
                for lay in layouts:
                    times[lay].append(time_ms(lay, reps))
            base = statistics.median(times["one-plain"])
            for lay in layouts:
                med = statistics.median(times[lay])
                lengths = layout_lengths(lay, S)
                rec = {"geometry": geo, "nh": nh, "nkv": nkv, "S": S, "layout": lay, "n_docs": len(lengths),
                       "ms_median": round(med, 4), "ms_min": round(min(times[lay]), 4),
                       "ms_max": round(max(times[lay]), 4),
                       "useful_tflops": round(useful_flop(lengths, nh) / med / 1e9, 1),
                       "speedup_vs_one_doc": round(base / med, 3)}
                out.append(rec)
                print(f"{geo:10s} S {S:5d} {lay:10s} {med:8.3f} ms  {rec['useful_tflops']:6.1f} TFLOP/s  "
                      f"x{rec['speedup_vs_one_doc']:.2f}", flush=True)
            del qkv, do
            torch.cuda.empty_cache()
    return out


def e2e_run(document_masking, steps, warmup):
    import torch

    from distributed_training_guide_b200.engine import TrainEngine

    S = 4096
    dev = torch.device("cuda", 0)
    eng = TrainEngine.create("meta-llama/Llama-2-7b-hf", parallelism="single", batch_size=1, seq_length=S,
                             device="cuda", document_masking=document_masking)
    batches = [eng.synthetic_batch(seed=i) for i in range(steps + warmup)]
    pos = positions(layout_lengths("docs512", S)).pin_memory()
    for b in batches:
        b["position_ids"] = pos
    for b in batches[:warmup]:
        loss = eng.step(b)
    torch.cuda.synchronize(dev)
    t0 = time.perf_counter()
    for b in batches[warmup:]:
        loss = eng.step(b)
    torch.cuda.synchronize(dev)
    ms = (time.perf_counter() - t0) * 1e3 / steps
    out = {"document_masking": document_masking, "ms_per_step": ms, "tokens_per_s": S / ms * 1e3, "loss": float(loss),
           "peak_alloc_gb": torch.cuda.max_memory_allocated(dev) / 1e9}
    eng.close()
    return out


def e2e_in_subprocess(document_masking, a):
    cmd = [sys.executable, __file__, "--e2e-one", "on" if document_masking else "off", "--steps", str(a.steps),
           "--warmup", str(a.warmup)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        return {"document_masking": document_masking, "error": (r.stdout + r.stderr).strip().splitlines()[-1]}
    return json.loads(r.stdout.strip().splitlines()[-1])


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--skip-e2e", action="store_true")
    ap.add_argument("--e2e-one", choices=("off", "on"), help=argparse.SUPPRESS)   # one end-to-end run, then exit
    a = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        sys.exit("bench_docmask.py measures on a CUDA device; none is visible")
    from distributed_training_guide_b200 import _ext

    _ext.load(required=True)
    if a.e2e_one:
        print(json.dumps(e2e_run(a.e2e_one == "on", a.steps, a.warmup)))
        return
    info = gpu_info()
    kernels = kernel_section(a.reps, a.rounds)
    e2e = [] if a.skip_e2e else [e2e_in_subprocess(dm, a) for dm in (False, True, False, True)]
    summary = {}
    for r in kernels:
        if r["layout"] == "one-doc":
            summary[f"{r['geometry']}_S{r['S']}_doc_over_plain_one_doc"] = round(r["ms_median"] / next(
                x["ms_median"] for x in kernels if x["geometry"] == r["geometry"] and x["S"] == r["S"]
                and x["layout"] == "one-plain"), 4)
        if r["layout"] == "docs512":
            summary[f"{r['geometry']}_S{r['S']}_docs512_speedup"] = r["speedup_vs_one_doc"]
    for dm in (False, True):
        vals = [r["ms_per_step"] for r in e2e if r.get("document_masking") == dm and "ms_per_step" in r]
        if vals:
            summary[f"e2e_ms_per_step_{'docmask' if dm else 'plain'}"] = round(statistics.mean(vals), 2)
    print(json.dumps({"gpu": info, "kernels": kernels, "e2e": e2e, "summary": summary}))


if __name__ == "__main__":
    main()
