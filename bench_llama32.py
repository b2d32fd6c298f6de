"""head_dim-64 attention on one H100: Llama-3.2-1B attention shapes and a Llama-3.2-1B training step, the D = 64
wgmma kernels against the SDPA path that head_dim-64 models took before those kernels existed.

    python bench_llama32.py [--reps 10] [--rounds 5] [--steps 5] [--warmup 2] [--skip-e2e]

Kernel section: B 1, 32 q heads : 8 kv heads, head_dim 64 (Llama-3.2-1B), S 4096 and 8192, forward alone (under
``no_grad``) and forward + backward (``torch.autograd.grad``).  Five cases per shape and pass:
- ``kernel``: ``ops.attention_qkv``, plain causal, on the D = 64 kernels;
- ``sdpa``: the same call routed to its SDPA fallback, with the backend SDPA picks itself (what training ran);
- ``sdpa-flash``: the same fallback with the flash backend forced (PyTorch's FA2);
- ``kernel-docs8``: 8 equal documents through the document-masking kernels;
- ``sdpa-docs8``: the same documents through the fallback, SDPA with the dense [1, 1, S, S] mask.
Cases alternate inside each round; the median over rounds is reported with TFLOP/s over the visible (q, k) pairs,
computed here (S(S+1)/2 causal, the sum of L(L+1)/2 over documents), and as a share of the 989 TFLOP/s dense BF16
data-sheet figure: attention at these shapes is compute-bound (about 2 * 64 FLOPs per loaded byte and key block).

End-to-end section: single-GPU ``TrainEngine`` steps of Llama-3.2-1B (S 4096, B 1), plain and with document masking
on 512-token documents, on the kernels and with ``DTG_FORCE_REFERENCE=attention`` (the SDPA fallback), each in a
process of its own, alternating.  Device-timed tokens/s and peak allocated memory.  The card's name and power limit
are read in the same run.  Prints one JSON record as the last line.
"""
from __future__ import annotations

import argparse
import contextlib
import json
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

NH, NKV, D, NDOCS = 32, 8, 64, 8
MODEL = "meta-llama/Llama-3.2-1B"
PEAK_TFLOPS = 989.0   # H100 SXM, dense BF16, data sheet


def gpu_info():
    q = ["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"]
    try:
        line = subprocess.run(q, capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, sm, sm_max = [s.strip() for s in line.split(",")]
        return {"name": name, "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max}
    except Exception as e:  # the numbers still stand, but without their card
        return {"error": repr(e)}


def visible_pairs(lengths):
    """Causal (q, k) pairs inside each document."""
    return sum(n * (n + 1) // 2 for n in lengths)


def flop(lengths, backward):
    """Matmul FLOPs over the visible pairs: QK^T and PV forward, plus QK^T again, dP, dV, dQ and dK backward."""
    return (7 if backward else 2) * 2 * D * NH * visible_pairs(lengths)


def kernel_section(reps, rounds):
    import torch
    from torch.nn.attention import SDPBackend, sdpa_kernel

    from distributed_training_guide_b200 import _ext, ops

    out = []
    for S in (4096, 8192):
        g = torch.Generator(device="cuda").manual_seed(0)
        qkv = torch.randn(1, S, NH + 2 * NKV, D, device="cuda", generator=g).to(torch.bfloat16).requires_grad_(True)
        do = torch.randn(1, S, NH, D, device="cuda", generator=g).to(torch.bfloat16)
        L = S // NDOCS
        ds = ops.document_starts((torch.arange(S) % L)[None].cuda())
        names = ("kernel", "sdpa", "sdpa-flash", "kernel-docs8", "sdpa-docs8")
        baselines = {"kernel": ("sdpa", "sdpa-flash"), "kernel-docs8": ("sdpa-docs8",)}
        cases = [(n, bwd) for bwd in (False, True) for n in names]
        forced = _ext._forced

        def run(name, bwd):
            docs = ds if name.endswith("docs8") else None
            _ext._forced = forced | {"attention"} if name.startswith("sdpa") else forced
            try:
                with sdpa_kernel(SDPBackend.FLASH_ATTENTION) if name == "sdpa-flash" else contextlib.nullcontext():
                    if bwd:
                        o = ops.attention_qkv(qkv, NH, NKV, doc_start=docs)
                        return torch.autograd.grad(o, qkv, do)
                    with torch.no_grad():
                        return ops.attention_qkv(qkv, NH, NKV, doc_start=docs)
            finally:
                _ext._forced = forced

        def time_ms(case, n):
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            for _ in range(n):
                run(*case)
            e.record()
            e.synchronize()
            return s.elapsed_time(e) / n

        # the kernel path must launch this project's kernels, the fallback none
        n0 = _ext.launch_count()
        run("kernel", True)
        torch.cuda.synchronize()
        assert _ext.launch_count() - n0 == 4, "the D = 64 kernels did not run"
        n0 = _ext.launch_count()
        for name in names[1:]:
            if name.startswith("sdpa"):
                run(name, True)
        torch.cuda.synchronize()
        assert _ext.launch_count() == n0, "the SDPA fallback launched a kernel of the extension"
        for c in cases:
            time_ms(c, 2)
        times = {c: [] for c in cases}
        for _ in range(rounds):
            for c in cases:
                times[c].append(time_ms(c, reps))
        for c in cases:
            name, bwd = c
            med = statistics.median(times[c])
            lengths = [L] * NDOCS if name.endswith("docs8") else [S]
            tf = flop(lengths, bwd) / med / 1e9
            rec = {"S": S, "nh": NH, "nkv": NKV, "head_dim": D, "case": name, "pass": "fwd+bwd" if bwd else "fwd",
                   "n_docs": len(lengths), "visible_pairs_per_head": visible_pairs(lengths),
                   "ms_median": round(med, 4), "ms_min": round(min(times[c]), 4), "ms_max": round(max(times[c]), 4),
                   "tflops_visible": round(tf, 1), "share_of_989_tflops": round(tf / PEAK_TFLOPS, 3),
                   "bound": "compute"}
            for other in baselines.get(name, ()):
                rec[f"speedup_vs_{other}"] = round(statistics.median(times[(other, bwd)]) / med, 3)
            out.append(rec)
            vs = "  ".join(f"x{v:.2f} vs {k[11:]}" for k, v in rec.items() if k.startswith("speedup_vs_"))
            print(f"S {S:5d} {rec['pass']:7s} {name:13s} {med:9.3f} ms  {tf:6.1f} TFLOP/s "
                  f"({rec['share_of_989_tflops']:.2f} of 989)  {vs}", flush=True)
        del qkv, do
        torch.cuda.empty_cache()
    return out


def e2e_run(document_masking, steps, warmup):
    import torch

    from distributed_training_guide_b200 import _ext
    from distributed_training_guide_b200.engine import TrainEngine

    S = 4096
    dev = torch.device("cuda", 0)
    eng = TrainEngine.create(MODEL, parallelism="single", batch_size=1, seq_length=S, device="cuda",
                             document_masking=document_masking)
    batches = [eng.synthetic_batch(seed=i) for i in range(steps + warmup)]
    if document_masking:
        pos = (torch.arange(S) % 512)[None].pin_memory()
        for b in batches:
            b["position_ids"] = pos
    for b in batches[:warmup]:
        loss = eng.step(b)
    torch.cuda.synchronize(dev)
    n0 = _ext.launch_count()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0 = time.perf_counter()
    s.record()
    for b in batches[warmup:]:
        loss = eng.step(b)
    e.record()
    torch.cuda.synchronize(dev)
    host_ms = (time.perf_counter() - t0) * 1e3 / steps
    dev_ms = s.elapsed_time(e) / steps
    out = {"model": MODEL, "attention": "sdpa" if "attention" in _ext._forced else "kernel",
           "document_masking": document_masking, "S": S, "B": 1, "ms_per_step_device": round(dev_ms, 2),
           "ms_per_step_host": round(host_ms, 2), "tokens_per_s_device": round(S / dev_ms * 1e3),
           "launches_per_step": (_ext.launch_count() - n0) // steps, "loss": float(loss),
           "peak_alloc_gb": round(torch.cuda.max_memory_allocated(dev) / 1e9, 2)}
    eng.close()
    return out


def e2e_in_subprocess(sdpa, document_masking, a):
    cmd = [sys.executable, __file__, "--e2e-one", "on" if document_masking else "off", "--steps", str(a.steps),
           "--warmup", str(a.warmup)]
    env = dict(os.environ)
    env.pop("DTG_FORCE_REFERENCE", None)
    if sdpa:
        env["DTG_FORCE_REFERENCE"] = "attention"
    r = subprocess.run(cmd, capture_output=True, text=True, env=env)
    if r.returncode != 0:
        sys.stderr.write((r.stdout + r.stderr)[-2000:])
        return {"attention": "sdpa" if sdpa else "kernel", "document_masking": document_masking,
                "error": (r.stdout + r.stderr).strip().splitlines()[-1]}
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
        sys.exit("bench_llama32.py measures on a CUDA device; none is visible")
    from distributed_training_guide_b200 import _ext

    _ext.load(required=True)
    if a.e2e_one:
        print(json.dumps(e2e_run(a.e2e_one == "on", a.steps, a.warmup)))
        return
    info = gpu_info()
    print(f"gpu: {info}", flush=True)
    kernels = kernel_section(a.reps, a.rounds)
    e2e = "not measured"
    if not a.skip_e2e:
        e2e = []
        for dm in (False, True):
            for sdpa in (False, True, False, True):
                e2e.append(e2e_in_subprocess(sdpa, dm, a))
                print(f"e2e: {e2e[-1]}", flush=True)
    summary = {}
    for r in kernels:
        for key in (k for k in r if k.startswith("speedup_vs_")):
            summary[f"S{r['S']}_{r['pass']}_{r['case']}_{key}"] = r[key]
    for dm in (False, True):
        for att in ("kernel", "sdpa"):
            vals = [r["tokens_per_s_device"] for r in (e2e if isinstance(e2e, list) else [])
                    if "tokens_per_s_device" in r and r["attention"] == att and r["document_masking"] == dm]
            summary[f"e2e_tokens_per_s_{att}{'_docs' if dm else ''}"] = round(statistics.mean(vals)) if vals \
                else "not measured"
    print(json.dumps({"gpu": info, "kernels": kernels, "e2e": e2e, "summary": summary}))


if __name__ == "__main__":
    main()
