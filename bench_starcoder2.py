"""StarCoder2's new kernels on one H100, and StarCoder2 training steps beside Llama-3.2-3B.

    python bench_starcoder2.py [--reps 20] [--rounds 5] [--steps 5] [--warmup 2] [--skip-e2e]

Kernel section, T 4096, at StarCoder2-3B, -7B and -15B shapes (hidden 3072 / 4608 / 6144, intermediate 12288 / 18432
/ 24576).  CUDA-event medians over rounds, the cases alternating inside each round, of
  * ``ln_fwd`` (``layernorm_fwd`` with a residual): reads x, r, w, b, writes h, y, mean and rstd; against
    ``aten_ln_fwd``, ATen's ``x + r`` then ``F.layer_norm``;
  * ``ln_bwd`` (``layernorm_bwd`` with ``dres``): reads dy, h, dres, w, mean, rstd, writes dx and the dw / db partial
    rows, which ``colsum`` reads back into dw and db; against ``aten_ln_bwd``, the autograd backward of
    ``F.layer_norm`` (plus the add of the residual gradient);
  * ``gelu_fwd`` / ``gelu_bwd`` on [4096, I]: against ATen's ``F.gelu(approximate="tanh")`` and its autograd backward.
The bytes each of our kernels has to move come from the shapes (the backward's partial rows from its grid); ATen's
cases are charged the same bytes, the least their operation needs.  GB/s is over the median time, and the share is of
the H100 SXM data-sheet bandwidth of 3.35 TB/s.

End-to-end section: device-timed single-GPU ``TrainEngine`` steps at S 4096, B 1 of bigcode/starcoder2-3b, its
neighbour meta-llama/Llama-3.2-3B, and bigcode/starcoder2-7b (whether it fits on one 80 GB card with its AdamW state),
each in a process of its own: ms/step, tokens/s and peak memory.  The card's name and power limit are read in the same
run.  Prints one JSON record as the last line.
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

MODELS = ("bigcode/starcoder2-3b", "meta-llama/Llama-3.2-3B", "bigcode/starcoder2-7b")
SHAPES = {"StarCoder2-3B": (3072, 12288), "StarCoder2-7B": (4608, 18432), "StarCoder2-15B": (6144, 24576)}
T, S, EPS = 4096, 4096, 1e-5
PEAK_BW = 3.35e12


def kernel_bytes(H, I, bwd_grid):
    row = T * H * 2
    vec = H * 2
    stats = 2 * T * 4
    partial = 2 * bwd_grid * H * 4
    act = T * I * 2
    return {
        # reads x and r, writes h and y; w, b; mean and rstd
        "ln_fwd": 4 * row + 2 * vec + stats,
        # reads dy, h and dres, writes dx; w; mean and rstd; the partials written and read back; dw and db
        "ln_bwd": 4 * row + vec + stats + 2 * partial + 2 * H * 4,
        "gelu_fwd": 2 * act,
        "gelu_bwd": 3 * act,
    }


def kernel_section(reps, rounds):
    import torch
    import torch.nn.functional as F

    from distributed_training_guide_b200 import _ext

    C = _ext.load(required=True)
    out = []

    def time_ms(fn, n):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(n):
            fn()
        e.record()
        e.synchronize()
        return s.elapsed_time(e) / n

    for shape, (H, I) in SHAPES.items():
        g = torch.Generator(device="cuda").manual_seed(0)
        x = torch.randn(T, H, device="cuda", generator=g).to(torch.bfloat16)
        r = torch.randn(T, H, device="cuda", generator=g).to(torch.bfloat16)
        dy = torch.randn(T, H, device="cuda", generator=g).to(torch.bfloat16)
        dres = torch.randn(T, H, device="cuda", generator=g).to(torch.bfloat16)
        w = (1 + 0.1 * torch.randn(H, device="cuda", generator=g)).to(torch.bfloat16)
        b = (0.1 * torch.randn(H, device="cuda", generator=g)).to(torch.bfloat16)
        _, h, mean, rstd = C.layernorm_fwd(x, r, w, b, EPS)
        u = torch.randn(T, I, device="cuda", generator=g).to(torch.bfloat16)
        du = torch.randn(T, I, device="cuda", generator=g).to(torch.bfloat16)
        ha = h.clone().requires_grad_()
        wa, ba = w.clone().requires_grad_(), b.clone().requires_grad_()
        ya = F.layer_norm(ha, (H,), wa, ba, EPS)
        ua = u.clone().requires_grad_()
        ga = F.gelu(ua, approximate="tanh")

        def aten_ln_bwd():
            dx, _, _ = torch.autograd.grad(ya, (ha, wa, ba), dy, retain_graph=True)
            return dx + dres

        cases = {
            "ln_fwd": lambda: C.layernorm_fwd(x, r, w, b, EPS),
            "aten_ln_fwd": lambda: F.layer_norm(x + r, (H,), w, b, EPS),
            "ln_bwd": lambda: C.layernorm_bwd(dy, h, w, mean, rstd, dres),
            "aten_ln_bwd": aten_ln_bwd,
            "gelu_fwd": lambda: C.gelu_tanh_fwd(u),
            "aten_gelu_fwd": lambda: F.gelu(u, approximate="tanh"),
            "gelu_bwd": lambda: C.gelu_tanh_bwd(du, u),
            "aten_gelu_bwd": lambda: torch.autograd.grad(ga, ua, du, retain_graph=True),
        }
        for fn in cases.values():
            time_ms(fn, 3)
        times = {k: [] for k in cases}
        for _ in range(rounds):
            for k, fn in cases.items():
                times[k].append(time_ms(fn, reps))
        nbytes = kernel_bytes(H, I, C.layernorm_bwd_grid(T, H))
        for k in cases:
            op = k.replace("aten_", "")
            med = statistics.median(times[k])
            gbs = nbytes[op] / (med * 1e-3) / 1e9
            rec = {"shape": shape, "op": k, "bytes": nbytes[op], "us_median": round(med * 1e3, 1),
                   "us_min": round(min(times[k]) * 1e3, 1), "us_max": round(max(times[k]) * 1e3, 1),
                   "GB_per_s": round(gbs, 1), "share_of_3.35TB_per_s": round(gbs * 1e9 / PEAK_BW, 3)}
            out.append(rec)
            print(f"{shape:15s} {k:14s} {med * 1e3:9.1f} us  {gbs:7.1f} GB/s  "
                  f"{rec['share_of_3.35TB_per_s']:.2f} of 3.35 TB/s", flush=True)
    return out


def e2e_run(model, steps, warmup):
    import torch

    from distributed_training_guide_b200.engine import TrainEngine

    dev = torch.device("cuda", 0)
    eng = TrainEngine.create(model, parallelism="single", batch_size=1, seq_length=S, device="cuda")
    batches = [eng.synthetic_batch(seed=i) for i in range(steps + warmup)]
    for bt in batches[:warmup]:
        loss = eng.step(bt)
    torch.cuda.synchronize(dev)
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0 = time.perf_counter()
    s.record()
    for bt in batches[warmup:]:
        loss = eng.step(bt)
    e.record()
    torch.cuda.synchronize(dev)
    host_ms = (time.perf_counter() - t0) * 1e3 / steps
    dev_ms = s.elapsed_time(e) / steps
    out = {"model": model, "S": S, "B": 1, "ms_per_step_device": round(dev_ms, 2), "ms_per_step_host": round(host_ms, 2),
           "tokens_per_s_device": round(S / dev_ms * 1e3), "loss": float(loss),
           "peak_alloc_gb": round(torch.cuda.max_memory_allocated(dev) / 1e9, 2)}
    eng.close()
    return out


def e2e_in_subprocess(model, a):
    cmd = [sys.executable, __file__, "--e2e-one", model, "--steps", str(a.steps), "--warmup", str(a.warmup)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write((r.stdout + r.stderr)[-2000:])
        return {"model": model, "error": (r.stdout + r.stderr).strip().splitlines()[-1]}
    return json.loads(r.stdout.strip().splitlines()[-1])


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--skip-e2e", action="store_true")
    ap.add_argument("--e2e-one", default=None, help=argparse.SUPPRESS)   # one end-to-end run of this model, then exit
    a = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        sys.exit("bench_starcoder2.py measures on a CUDA device; none is visible")
    from distributed_training_guide_b200 import _ext

    _ext.load(required=True)
    if a.e2e_one:
        print(json.dumps(e2e_run(a.e2e_one, a.steps, a.warmup)))
        return
    info = gpu_info()
    print(f"gpu: {info}", flush=True)
    kernels = kernel_section(a.reps, a.rounds)
    e2e = "not measured"
    if not a.skip_e2e:
        e2e = []
        for model in MODELS:
            rec = e2e_in_subprocess(model, a)
            rec["fits_on_one_80GB_card"] = "error" not in rec
            print(f"e2e: {rec}", flush=True)
            e2e.append(rec)
    print(json.dumps({"gpu": info, "kernels": kernels, "e2e": e2e}))


if __name__ == "__main__":
    main()
