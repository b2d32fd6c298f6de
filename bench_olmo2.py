"""OLMo 2's two new kernels on one H100, and an OLMo-2-7B training step beside Llama-2-7B.

    python bench_olmo2.py [--reps 20] [--rounds 5] [--steps 5] [--warmup 2] [--layers N] [--skip-e2e]

Kernel section, B 1, S 4096, head_dim 128, at OLMo-2-7B shapes (32 q : 32 kv heads, hidden 4096) and OLMo-2-32B
shapes (40 : 8, hidden 5120).  CUDA-event medians over rounds, the cases alternating inside each round, of
  * ``full_fwd`` (``qk_norm_full_rope_fwd``): reads q|k and the cos/sin tables, writes q|k, the saved pre-norm q|k
    and two rstd per token;
  * ``full_bwd`` (``qk_norm_full_rope_bwd``): reads dq|dk, the saved q|k, the rstd, the gains and the tables, writes
    dq|dk, the per-CTA gain-gradient partials and (``colsum``) their sum, which it reads back;
  * ``unfused``: ATen ``rms_norm`` on the [S, nh*128] q and [S, nkv*128] k views, a copy back into the qkv buffer,
    then ``rope_inplace``;
  * ``rope_inplace`` alone (what a Llama layer runs there);
  * ``norm_add`` (``rmsnorm_add_fwd``) against ``rmsnorm_then_add`` (``rmsnorm_fwd`` then a bf16 ATen add) on
    [S, hidden].
The bytes each case has to move come from the shapes (the backward's partial rows from its grid); GB/s is over the
median time, and the share is of the H100 SXM data-sheet bandwidth of 3.35 TB/s.

End-to-end section: device-timed tokens/s of single-GPU ``TrainEngine`` steps of allenai/OLMo-2-1124-7B and of
meta-llama/Llama-2-7b-hf at S 4096, B 1, each in a process of its own.  When a model does not fit, it runs again
with ``--layers`` decoder layers and the record says so.  The card's name and power limit are read in the same run.
Prints one JSON record as the last line.
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

MODELS = ("allenai/OLMo-2-1124-7B", "meta-llama/Llama-2-7b-hf")
SHAPES = {"OLMo-2-7B": (32, 32, 4096), "OLMo-2-32B": (40, 8, 5120)}   # nh, nkv, hidden
S, D, EPS = 4096, 128, 1e-6
PEAK_BW = 3.35e12


def kernel_bytes(nh, nkv, hidden, bwd_grid):
    qk = S * (nh + nkv) * D * 2           # the q|k heads in bf16
    gains = (nh + nkv) * D * 2
    tables = 2 * S * (D // 2) * 4
    rstd = S * 2 * 4
    partial = bwd_grid * (nh + nkv) * D * 4
    row = S * hidden * 2
    return {
        "full_fwd": 3 * qk + gains + tables + rstd,
        "full_bwd": 3 * qk + gains + tables + rstd + 2 * partial + (nh + nkv) * D * 4,
        # rms_norm reads x, writes y (q and k); the copy reads y and writes q|k; rope reads and writes q|k
        "unfused": 2 * qk + 2 * qk + 2 * qk + tables,
        "rope_inplace": 2 * qk + tables,
        # reads x and r, writes h (and rstd)
        "norm_add": 3 * row + S * 4,
        # rmsnorm_fwd reads x, writes y and rstd; the add reads y and r and writes h
        "rmsnorm_then_add": 2 * row + S * 4 + 3 * row,
    }


def kernel_section(reps, rounds):
    import torch

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

    for shape, (nh, nkv, hidden) in SHAPES.items():
        g = torch.Generator(device="cuda").manual_seed(0)
        qkv = torch.randn(1, S, nh + 2 * nkv, D, device="cuda", generator=g).to(torch.bfloat16)
        dqkv = torch.randn(1, S, nh + 2 * nkv, D, device="cuda", generator=g).to(torch.bfloat16)
        q_w = (1 + 0.1 * torch.randn(nh * D, device="cuda", generator=g)).to(torch.bfloat16)
        k_w = (1 + 0.1 * torch.randn(nkv * D, device="cuda", generator=g)).to(torch.bfloat16)
        cos, sin = ref.rope_tables(torch.arange(S, device="cuda"), D, 5e5)
        x_save, rstd = C.qk_norm_full_rope_fwd(qkv, q_w, k_w, cos, sin, nh, nkv, EPS)
        x = torch.randn(S, hidden, device="cuda", generator=g).to(torch.bfloat16)
        r = torch.randn(S, hidden, device="cuda", generator=g).to(torch.bfloat16)
        w = (1 + 0.1 * torch.randn(hidden, device="cuda", generator=g)).to(torch.bfloat16)
        qv = qkv[0, :, :nh].reshape(S, nh * D)
        kv = qkv[0, :, nh:nh + nkv].reshape(S, nkv * D)

        def unfused():
            q = torch.nn.functional.rms_norm(qv, (nh * D,), q_w, EPS)
            k = torch.nn.functional.rms_norm(kv, (nkv * D,), k_w, EPS)
            qkv[:, :, :nh].copy_(q.view(1, S, nh, D))
            qkv[:, :, nh:nh + nkv].copy_(k.view(1, S, nkv, D))
            C.rope_inplace(qkv, cos, sin, nh + nkv, False)

        def rmsnorm_then_add():
            y, _, _ = C.rmsnorm_fwd(x, w, EPS, None)
            return r + y

        # every case works in place on buffers whose values stay in range when it is repeated (normalised heads)
        cases = {
            "full_fwd": lambda: C.qk_norm_full_rope_fwd(qkv, q_w, k_w, cos, sin, nh, nkv, EPS),
            "full_bwd": lambda: C.qk_norm_full_rope_bwd(dqkv, x_save, rstd, q_w, k_w, cos, sin, nh, nkv),
            "unfused": unfused,
            "rope_inplace": lambda: C.rope_inplace(qkv, cos, sin, nh + nkv, False),
            "norm_add": lambda: C.rmsnorm_add_fwd(x, r, w, EPS),
            "rmsnorm_then_add": rmsnorm_then_add,
        }
        for fn in cases.values():
            time_ms(fn, 3)
        times = {k: [] for k in cases}
        for _ in range(rounds):
            for k, fn in cases.items():
                times[k].append(time_ms(fn, reps))
        grid = C.qk_norm_full_rope_bwd_grid(S, nh + nkv)
        nbytes = kernel_bytes(nh, nkv, hidden, grid)
        for k in cases:
            med = statistics.median(times[k])
            gbs = nbytes[k] / (med * 1e-3) / 1e9
            rec = {"shape": shape, "op": k, "bytes": nbytes[k], "ms_median": round(med, 4),
                   "ms_min": round(min(times[k]), 4), "ms_max": round(max(times[k]), 4), "GB_per_s": round(gbs, 1),
                   "share_of_3.35TB_per_s": round(gbs * 1e9 / PEAK_BW, 3)}
            out.append(rec)
            print(f"{shape:11s} {k:18s} {med * 1e3:9.1f} us  {gbs:7.1f} GB/s  "
                  f"{rec['share_of_3.35TB_per_s']:.2f} of 3.35 TB/s", flush=True)
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
    ap.add_argument("--layers", type=int, default=0, help="decoder layers for a step when the whole model does not fit")
    ap.add_argument("--skip-e2e", action="store_true")
    ap.add_argument("--e2e-one", default=None, help=argparse.SUPPRESS)   # one end-to-end run of this model, then exit
    a = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        sys.exit("bench_olmo2.py measures on a CUDA device; none is visible")
    from distributed_training_guide_b200 import _ext

    _ext.load(required=True)
    if a.e2e_one:
        print(json.dumps(e2e_run(a.e2e_one, a.layers, a.steps, a.warmup)))
        return
    info = gpu_info()
    print(f"gpu: {info}", flush=True)
    kernels = kernel_section(a.reps, a.rounds)
    e2e = "not measured"
    if not a.skip_e2e:
        e2e = []
        for model in MODELS:
            rec = e2e_in_subprocess(model, 0, a)
            print(f"e2e: {rec}", flush=True)
            if "error" in rec:
                rec["fits_in_80GB"] = False
                e2e.append(rec)
                rec = e2e_in_subprocess(model, a.layers or 16, a)
                print(f"e2e (reduced to {a.layers or 16} layers): {rec}", flush=True)
            e2e.append(rec)
    print(json.dumps({"gpu": info, "kernels": kernels, "e2e": e2e}))


if __name__ == "__main__":
    main()
