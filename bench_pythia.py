"""GPT-NeoX's new kernels on one H100, and Pythia training steps.

    python bench_pythia.py [--reps 20] [--rounds 5] [--steps 5] [--warmup 2] [--skip-e2e]

Kernel section, T 2048 (S 2048, B 1), at Pythia-1.4B and -6.9B shapes (hidden 2048 / 4096, intermediate 8192 / 16384,
16 / 32 heads of 128, rotary 32).  CUDA-event medians over rounds, the cases alternating inside each round, of
  * ``ln2_fwd`` (``layernorm2_fwd`` with a residual): reads x, r, two gains and biases, writes h, y1, y2, mean and
    rstd; against ``add_ln+ln``, this project's ``layernorm_fwd`` with the residual, then again on h without it (what
    two separate norms of one stream cost);
  * ``ln2_bwd`` (``layernorm2_bwd`` with ``dres``): reads dy1, dy2, h, dres, writes dx and four partial rows per CTA
    that ``colsum`` reads back; against ``ln_bwd x2``, two ``layernorm_bwd`` calls, the second taking the first's dx
    as its residual gradient;
  * ``rope_partial`` (``rope_inplace`` with rot_dim 32 on the q and k heads, in place): against ``aten_rope_partial``,
    ``ref.rope_apply`` on the slice and a copy back;
  * ``gelu_fwd`` / ``gelu_bwd`` (exact) on [2048, I]: against ATen's ``F.gelu`` and its autograd backward.
The bytes each of our kernels has to move come from the shapes (the backward's partial rows from its grid); the
unfused cases are charged their own bytes, ATen's the bytes of our kernel.  GB/s is over the median time, and the
share is of the H100 SXM data-sheet bandwidth of 3.35 TB/s.

End-to-end section: device-timed single-GPU ``TrainEngine`` steps at S 2048, B 1 of EleutherAI/pythia-1.4b and
EleutherAI/pythia-6.9b, each in a process of its own: ms/step, tokens/s and peak memory.  The card's name and power
limit are read in the same run.  Prints one JSON record as the last line.
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

MODELS = ("EleutherAI/pythia-1.4b", "EleutherAI/pythia-6.9b")
SHAPES = {"Pythia-1.4B": (2048, 8192, 16), "Pythia-6.9B": (4096, 16384, 32)}   # hidden, intermediate, heads
T, S, D, ROT, EPS = 2048, 2048, 128, 32, 1e-5
PEAK_BW = 3.35e12


def kernel_bytes(H, I, nh, ln_grid, ln2_grid):
    row, vec, stats = T * H * 2, H * 2, 2 * T * 4
    act = T * I * 2
    rope = 2 * (T * 2 * nh * ROT * 2) + 2 * S * (ROT // 2) * 4   # q|k slices read and written; cos, sin
    return {
        "ln2_fwd": 5 * row + 4 * vec + stats,                       # x, r in; h, y1, y2 out
        # dy1, dy2, h, dres in, dx out (h read twice from L2 is not charged); the partials written and read back
        "ln2_bwd": 5 * row + 2 * vec + stats + 2 * 4 * ln2_grid * H * 4 + 4 * H * 4,
        "add_ln+ln": (4 * row + 2 * vec + stats) + (2 * row + 2 * vec + stats),
        "ln_bwd x2": 2 * (4 * row + vec + stats + 2 * 2 * ln_grid * H * 4 + 2 * H * 4),
        "rope_partial": rope,
        "gelu_fwd": 2 * act,
        "gelu_bwd": 3 * act,
    }


def kernel_section(reps, rounds):
    import torch
    import torch.nn.functional as F

    from distributed_training_guide_b200 import _ext
    from distributed_training_guide_b200.ops import reference as ref

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

    for shape, (H, I, nh) in SHAPES.items():
        g = torch.Generator(device="cuda").manual_seed(0)

        def rnd(*sh, scale=1.0, shift=0.0):
            return (shift + scale * torch.randn(*sh, device="cuda", generator=g)).to(torch.bfloat16)

        x, r, dy1, dy2, dres = (rnd(T, H) for _ in range(5))
        w1, w2 = rnd(H, scale=0.1, shift=1.0), rnd(H, scale=0.1, shift=1.0)
        b1, b2 = rnd(H, scale=0.1), rnd(H, scale=0.1)
        _, _, h, mean, rstd = C.layernorm2_fwd(x, r, w1, b1, w2, b2, EPS)
        qkv = rnd(1, S, 3 * nh, D)
        cos, sin = ref.rope_tables(torch.arange(S, device="cuda"), ROT, 1e4)
        u, du = rnd(T, I), rnd(T, I)
        ua = u.clone().requires_grad_()
        ga = F.gelu(ua)

        def unfused_fwd():
            _, hh, _, _ = C.layernorm_fwd(x, r, w1, b1, EPS)
            return C.layernorm_fwd(hh, None, w2, b2, EPS)

        def unfused_bwd():
            dx1, _, _ = C.layernorm_bwd(dy1, h, w1, mean, rstd, dres)
            return C.layernorm_bwd(dy2, h, w2, mean, rstd, dx1)

        def aten_rope():
            qk = qkv[:, :, :2 * nh, :ROT]
            qkv[:, :, :2 * nh, :ROT] = ref.rope_apply(qk, cos, sin)

        cases = {
            "ln2_fwd": lambda: C.layernorm2_fwd(x, r, w1, b1, w2, b2, EPS),
            "add_ln+ln": unfused_fwd,
            "ln2_bwd": lambda: C.layernorm2_bwd(dy1, dy2, h, w1, w2, mean, rstd, dres),
            "ln_bwd x2": unfused_bwd,
            "rope_partial": lambda: C.rope_inplace(qkv, cos, sin, 2 * nh, False, rot_dim=ROT),
            "aten_rope_partial": aten_rope,
            "gelu_fwd": lambda: C.gelu_fwd(u),
            "aten_gelu_fwd": lambda: F.gelu(u),
            "gelu_bwd": lambda: C.gelu_bwd(du, u),
            "aten_gelu_bwd": lambda: torch.autograd.grad(ga, ua, du, retain_graph=True),
        }
        for fn in cases.values():
            time_ms(fn, 3)
        times = {k: [] for k in cases}
        for _ in range(rounds):
            for k, fn in cases.items():
                times[k].append(time_ms(fn, reps))
        nbytes = kernel_bytes(H, I, nh, C.layernorm_bwd_grid(T, H), C.layernorm2_bwd_grid(T, H))
        for k in cases:
            op = k.replace("aten_", "")
            med = statistics.median(times[k])
            gbs = nbytes[op] / (med * 1e-3) / 1e9
            rec = {"shape": shape, "op": k, "bytes": nbytes[op], "us_median": round(med * 1e3, 1),
                   "us_min": round(min(times[k]) * 1e3, 1), "us_max": round(max(times[k]) * 1e3, 1),
                   "GB_per_s": round(gbs, 1), "share_of_3.35TB_per_s": round(gbs * 1e9 / PEAK_BW, 3)}
            out.append(rec)
            print(f"{shape:12s} {k:18s} {med * 1e3:9.1f} us  {gbs:7.1f} GB/s  "
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
        sys.exit("bench_pythia.py measures on a CUDA device; none is visible")
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
            print(f"e2e: {rec}", flush=True)
            e2e.append(rec)
    print(json.dumps({"gpu": info, "kernels": kernels, "e2e": e2e}))


if __name__ == "__main__":
    main()
