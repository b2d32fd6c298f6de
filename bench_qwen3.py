"""QK-norm + RoPE on one H100: the fused kernels at Qwen3-8B shapes, and a Qwen3-8B training step.

    python bench_qwen3.py [--reps 20] [--rounds 5] [--steps 5] [--warmup 2] [--layers N] [--skip-e2e]

Kernel section: B 1, S 4096, 32 q heads : 8 kv heads, head_dim 128 (Qwen3-8B).  CUDA-event medians over rounds, the
cases alternating inside each round, of
  * ``qk_norm_rope_fwd``: reads q|k and the cos/sin tables, writes q|k, the saved pre-norm q|k and rstd;
  * ``qk_norm_rope_bwd``: reads dq|dk, the saved q|k, rstd and the tables, writes dq|dk (the per-CTA gain partials
    and their reduction are counted too);
  * ``rope_inplace`` alone (what a Llama layer runs there): reads and writes q|k;
  * the unfused composition: ``ref.rms_norm`` (ATen) on the q and the k heads, a copy back into the qkv buffer and
    ``rope_inplace``.
The bytes each kernel has to move come from the shapes; GB/s is over the median time, and the share is of the H100
SXM data-sheet bandwidth of 3.35 TB/s.

End-to-end section: the device-timed tokens/s of single-GPU ``TrainEngine`` steps of Qwen/Qwen3-8B at S 4096, B 1,
in a process of its own.  When the whole model does not fit (its weights, gradients and AdamW state alone take about
65 GB), it runs again with ``--layers`` of its 36 decoder layers and the record says so.  The card's name and power
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

MODEL = "Qwen/Qwen3-8B"
S, NH, NKV, D, EPS = 4096, 32, 8, 128, 1e-6
PEAK_BW = 3.35e12


def kernel_bytes():
    qk = S * (NH + NKV) * D * 2          # the q|k heads in bf16
    tables = 2 * S * (D // 2) * 4
    rstd = S * (NH + NKV) * 4
    return {
        "qk_norm_rope_fwd": 3 * qk + tables + rstd,
        "qk_norm_rope_bwd": 3 * qk + tables + rstd,
        "rope_inplace": 2 * qk + tables,
        # rms_norm reads x, writes y (q and k); the copy reads y and writes q|k; rope reads and writes q|k
        "unfused_rmsnorm_copy_rope": 2 * qk + 2 * qk + 2 * qk + tables,
    }


def kernel_section(reps, rounds):
    import torch

    from distributed_training_guide_b200 import _ext
    from distributed_training_guide_b200.ops import reference as ref

    C = _ext.load(required=True)
    g = torch.Generator(device="cuda").manual_seed(0)
    qkv = torch.randn(1, S, NH + 2 * NKV, D, device="cuda", generator=g).to(torch.bfloat16)
    dqkv = torch.randn(1, S, NH + 2 * NKV, D, device="cuda", generator=g).to(torch.bfloat16)
    q_w = (1 + 0.1 * torch.randn(D, device="cuda", generator=g)).to(torch.bfloat16)
    k_w = (1 + 0.1 * torch.randn(D, device="cuda", generator=g)).to(torch.bfloat16)
    cos, sin = ref.rope_tables(torch.arange(S, device="cuda"), D, 1e6)
    x_save, rstd = C.qk_norm_rope_fwd(qkv, q_w, k_w, cos, sin, NH, NKV, EPS)

    def unfused():
        q = ref.rms_norm(qkv[:, :, :NH], q_w, EPS)
        k = ref.rms_norm(qkv[:, :, NH:NH + NKV], k_w, EPS)
        qkv[:, :, :NH].copy_(q)
        qkv[:, :, NH:NH + NKV].copy_(k)
        C.rope_inplace(qkv, cos, sin, NH + NKV, False)

    # every case works in place on buffers whose values stay in range when it is repeated (normalised heads)
    cases = {
        "qk_norm_rope_fwd": lambda: C.qk_norm_rope_fwd(qkv, q_w, k_w, cos, sin, NH, NKV, EPS),
        "qk_norm_rope_bwd": lambda: C.qk_norm_rope_bwd(dqkv, x_save, rstd, q_w, k_w, cos, sin, NH, NKV),
        "rope_inplace": lambda: C.rope_inplace(qkv, cos, sin, NH + NKV, False),
        "unfused_rmsnorm_copy_rope": unfused,
    }

    def time_ms(fn, n):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(n):
            fn()
        e.record()
        e.synchronize()
        return s.elapsed_time(e) / n

    for fn in cases.values():
        time_ms(fn, 3)
    times = {k: [] for k in cases}
    for _ in range(rounds):
        for k, fn in cases.items():
            times[k].append(time_ms(fn, reps))
    nbytes = kernel_bytes()
    out = []
    for k in cases:
        med = statistics.median(times[k])
        gbs = nbytes[k] / (med * 1e-3) / 1e9
        rec = {"op": k, "bytes": nbytes[k], "ms_median": round(med, 4), "ms_min": round(min(times[k]), 4),
               "ms_max": round(max(times[k]), 4), "GB_per_s": round(gbs, 1),
               "share_of_3.35TB_per_s": round(gbs * 1e9 / PEAK_BW, 3)}
        out.append(rec)
        print(f"{k:28s} {med * 1e3:9.1f} us  {gbs:7.1f} GB/s  {rec['share_of_3.35TB_per_s']:.2f} of 3.35 TB/s",
              flush=True)
    return out


def e2e_run(layers, steps, warmup):
    import torch

    from distributed_training_guide_b200.engine import TrainEngine

    dev = torch.device("cuda", 0)
    kw = {"num_layers": layers} if layers else {}
    eng = TrainEngine.create(MODEL, parallelism="single", batch_size=1, seq_length=S, device="cuda", **kw)
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
    out = {"model": MODEL, "num_layers": layers or eng.config.num_hidden_layers, "S": S, "B": 1,
           "ms_per_step_device": round(dev_ms, 2), "ms_per_step_host": round(host_ms, 2),
           "tokens_per_s_device": round(S / dev_ms * 1e3), "loss": float(loss),
           "peak_alloc_gb": round(torch.cuda.max_memory_allocated(dev) / 1e9, 2)}
    eng.close()
    return out


def e2e_in_subprocess(layers, a):
    cmd = [sys.executable, __file__, "--e2e-one", "--steps", str(a.steps), "--warmup", str(a.warmup),
           "--layers", str(layers)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write((r.stdout + r.stderr)[-2000:])
        return {"num_layers": layers or 36, "error": (r.stdout + r.stderr).strip().splitlines()[-1]}
    return json.loads(r.stdout.strip().splitlines()[-1])


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--layers", type=int, default=0, help="decoder layers for the step when all 36 do not fit")
    ap.add_argument("--skip-e2e", action="store_true")
    ap.add_argument("--e2e-one", action="store_true", help=argparse.SUPPRESS)   # one end-to-end run, then exit
    a = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        sys.exit("bench_qwen3.py measures on a CUDA device; none is visible")
    from distributed_training_guide_b200 import _ext

    _ext.load(required=True)
    if a.e2e_one:
        print(json.dumps(e2e_run(a.layers, a.steps, a.warmup)))
        return
    info = gpu_info()
    print(f"gpu: {info}", flush=True)
    kernels = kernel_section(a.reps, a.rounds)
    e2e = "not measured"
    if not a.skip_e2e:
        e2e = [e2e_in_subprocess(0, a)]
        print(f"e2e: {e2e[-1]}", flush=True)
        if "error" in e2e[-1]:
            e2e[-1]["fits_in_80GB"] = False
            e2e.append(e2e_in_subprocess(a.layers or 18, a))
            print(f"e2e (reduced to {a.layers or 18} layers): {e2e[-1]}", flush=True)
    print(json.dumps({"gpu": info, "kernels": kernels, "e2e": e2e}))


if __name__ == "__main__":
    main()
