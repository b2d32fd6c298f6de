"""Cost of gradient clipping (``--max-grad-norm``) on H100s.

    python bench_clip.py [--steps 10] [--warmup 3] [--seq-length 4096] [--skip-e2e]

Kernel section: on one bucket of Llama-2-7B decoder-layer size (202 M elements), the reduce + sum-of-squares kernel
of backward (one rank: reads and writes the bf16 gradient, 4 B per element) and the clipped AdamW kernel of
``optimizer.step()`` (bf16 parameters, gradient and moments: 14 B per element), timed with CUDA events, in GB/s and
as a fraction of the H100 SXM data-sheet 3.35 TB/s.

End-to-end section: ``TrainEngine`` on one GPU, Llama-2-7B, S 4096, B 1, without and with ``max_grad_norm=1.0``, in
alternating runs (off, on, off, on), each in a process of its own so that exactly one engine holds device memory.
Each step is timed on the device with CUDA events.  With two or more GPUs the same pair runs for ZeRO-1
(``parallelism="ddp"``) over every visible GPU.

The card's name and power limit are read in the same run.  Prints one JSON record as the last line.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

HBM_GBPS = 3350.0  # H100 SXM data sheet
LAYER_ELEMS = 202_383_360  # one Llama-2-7B decoder layer: 4*4096^2 + 3*4096*11008 + 2*4096


def gpu_info():
    q = ["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"]
    try:
        line = subprocess.run(q, capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, sm, sm_max = [s.strip() for s in line.split(",")]
        return {"name": name, "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max}
    except Exception as e:  # the numbers below still stand, but without their card
        return {"name": torch.cuda.get_device_name(), "error": repr(e)}


def _time_ms(fn, reps):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fn()
    torch.cuda.synchronize()
    s.record()
    for _ in range(reps):
        fn()
    e.record()
    e.synchronize()
    return s.elapsed_time(e) / reps


def kernel_section(reps, rounds):
    from distributed_training_guide_b200.parallel.symm import SymmGroup

    dev = torch.device("cuda", 0)
    sg = SymmGroup(dev, ranks=[0])
    n = LAYER_ELEMS
    try:
        gbuf, pbuf = sg.alloc(n, torch.bfloat16), sg.alloc(n, torch.bfloat16)
        gbuf.local.copy_(1e-3 * torch.randn(n, device=dev))
        pbuf.local.copy_(2e-2 * torch.randn(n, device=dev))
        m = torch.zeros(n, dtype=torch.bfloat16, device=dev)
        v = torch.zeros(n, dtype=torch.bfloat16, device=dev)
        ranges = torch.tensor([[0, n]], dtype=torch.int64, device=dev)
        partials = torch.zeros(sg.comm_blocks, dtype=torch.float64, device=dev)
        slots = sg.alloc(2, torch.float64)
        out = torch.zeros(2, dtype=torch.float32, device=dev)
        sg.clip_finalize_(partials, slots, 0, 1.0, 1.0, out)
        coef = out[1:]
        norm = lambda: sg.reduce_sumsq_(gbuf, 0, n, 1.0, False, ranges, partials)  # noqa: E731
        adamw = lambda: sg.C.comm_adamw_clip([pbuf.ptrs[0]], 0, pbuf.local, gbuf.local, m, v, 1e-5, 0.9, 0.999,  # noqa: E731
                                             1e-8, 0.01, 1, 1.0, coef)
        times = {"reduce_sumsq": [], "adamw_clip": []}
        for _ in range(rounds):
            times["reduce_sumsq"].append(_time_ms(norm, reps))
            times["adamw_clip"].append(_time_ms(adamw, reps))
        sg.check()
        rows = []
        for name, bytes_per in (("reduce_sumsq", 4), ("adamw_clip", 14)):
            ms = statistics.median(times[name])
            gbps = bytes_per * n / ms / 1e6
            rows.append({"kernel": name, "elements": n, "bytes_per_element": bytes_per, "ms": ms, "gbps": gbps,
                         "of_hbm_peak": gbps / HBM_GBPS})
        return rows
    finally:
        sg.close()


def e2e_run(clip, steps, warmup, seq, batch, parallelism):
    from distributed_training_guide_b200.engine import TrainEngine

    eng = TrainEngine.create("meta-llama/Llama-2-7b-hf", parallelism=parallelism, batch_size=batch, seq_length=seq,
                             max_grad_norm=1.0 if clip else None)
    dev = eng.device
    batches = [eng.synthetic_batch(seed=i) for i in range(steps + warmup)]
    for b in batches[:warmup]:
        loss = eng.step(b)
    torch.cuda.synchronize(dev)
    events = [torch.cuda.Event(enable_timing=True) for _ in range(steps + 1)]
    events[0].record()
    for i, b in enumerate(batches[warmup:]):
        loss = eng.step(b)
        events[i + 1].record()
    torch.cuda.synchronize(dev)
    step_ms = [events[i].elapsed_time(events[i + 1]) for i in range(steps)]
    out = {"parallelism": parallelism, "clip": clip, "world": eng.strategy.dp_size,
           "ms_per_step": statistics.mean(step_ms), "ms_per_step_median": statistics.median(step_ms),
           "tokens_per_s": eng.tokens_per_step / statistics.mean(step_ms) * 1e3, "loss": float(loss),
           "grad_norm": float(eng.grad_norm()) if clip else None,
           "peak_alloc_gb": torch.cuda.max_memory_allocated(dev) / 1e9}
    eng.close()
    return out


def e2e_in_subprocess(clip, a, nproc):
    args = [__file__, "--e2e-one", "on" if clip else "off", "--steps", str(a.steps), "--warmup", str(a.warmup),
            "--seq-length", str(a.seq_length), "--batch-size", str(a.batch_size)]
    if nproc > 1:
        cmd = [sys.executable, "-m", "torch.distributed.run", "--standalone", f"--nproc-per-node={nproc}", *args,
               "--parallelism", "ddp"]
    else:
        cmd = [sys.executable, *args, "--parallelism", "single"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    lines = [ln for ln in r.stdout.strip().splitlines() if ln.startswith("{")]
    if r.returncode != 0 or not lines:
        sys.stderr.write(r.stdout + r.stderr)
        return {"clip": clip, "world": nproc, "error": ((r.stdout + r.stderr).strip().splitlines() or ["?"])[-1]}
    return json.loads(lines[-1])


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--seq-length", type=int, default=4096)
    ap.add_argument("--batch-size", type=int, default=1)
    ap.add_argument("--skip-e2e", action="store_true")
    ap.add_argument("--e2e-one", choices=("off", "on"), help=argparse.SUPPRESS)   # one end-to-end run, then exit
    ap.add_argument("--parallelism", default="single", help=argparse.SUPPRESS)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_clip.py measures on a CUDA device; none is visible")
    if a.e2e_one:
        r = e2e_run(a.e2e_one == "on", a.steps, a.warmup, a.seq_length, a.batch_size, a.parallelism)
        if int(os.environ.get("RANK", "0")) == 0:
            print(json.dumps(r), flush=True)
        return
    info = gpu_info()
    print(f"# {info}", flush=True)
    rows = kernel_section(a.reps, a.rounds)
    for r in rows:
        print("# " + json.dumps(r), flush=True)
    e2e, summary = [], {}
    if not a.skip_e2e:
        ngpu = torch.cuda.device_count()
        for nproc in ([1, ngpu] if ngpu >= 2 else [1]):
            for clip in (False, True, False, True):
                r = e2e_in_subprocess(clip, a, nproc)
                print("# " + json.dumps(r), flush=True)
                e2e.append(r)
            key = "single" if nproc == 1 else f"zero1_x{nproc}"
            for clip in (False, True):
                vals = [r["ms_per_step"] for r in e2e if r.get("world") == nproc and r["clip"] == clip
                        and "ms_per_step" in r]
                if vals:
                    summary[f"{key}_{'clip' if clip else 'off'}_ms_per_step"] = statistics.mean(vals)
        if ngpu < 2:
            summary["zero1"] = "not measured: one GPU visible"
    print(json.dumps({"gpu": info, "kernels": rows, "e2e": e2e, "summary": summary}))


if __name__ == "__main__":
    main()
