"""Headline benchmark: training tokens/s of Llama-2-7B, seq 4096, bf16, on N H100s of one node —
DDP + ZeRO-1 for N > 1 (chapter 02's configuration), one process per GPU.

    python bench.py --gpus 1 --steps 5 --warmup 3
    python bench.py --gpus 1 --steps 5 --warmup 3 --dump-outputs /tmp/out   # + what the last timed step computed
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 8 --master-addr 127.0.0.1 \
        --master-port 29533 bench.py --gpus 8 --steps 5 --warmup 3

Protocol: W untimed warm-up steps, then K steps bracketed by barrier + cuda.synchronize, timed
with CUDA events on the device, max over ranks.  Two timed regions:
  * ``value``  — device-timed step loop with the batch already resident on the GPU;
  * ``e2e``    — the same K steps through the public API (``TrainEngine.step``) with, every step, the
                 host->device copy of that step's tokens from pinned memory and a device->host read
                 of the loss.
Synthetic tokens, random-init weights (seeded: the same arguments give the same inputs on every run).
Rank 0 prints ONE JSON line.

``--dump-outputs DIR`` (rank 0) writes, after the device-timed steps, what the last of them computed:
``loss.npy`` (the value ``TrainEngine.step`` returned, float32) and ``params_sample.npy`` (float32: the updated
weights at a fixed, seeded sample of up to 4096 positions per parameter, parameters in name order), so that two
builds of the project can be compared output for output.  It needs an engine whose every rank holds the full
parameters (one GPU, or ``--parallelism ddp``).
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

METRIC = "tokens/sec (device-timed, max over ranks) Llama-2-7B seq 4096 bf16 training"
PARALLELISM_NAMES = {"ddp": "dp", "fsdp": "fsdp", "tp": "tp", "2d": "fsdp_x_tp", "single": "single"}


class ClockSampler:
    """Samples SM clocks / throttle reasons of one GPU during the timed region (NVML)."""

    def __init__(self, index: int, period_s: float = 0.2):
        self.index, self.period = index, period_s
        self.samples, self.reasons, self.max_mhz = [], set(), None
        self._stop = threading.Event()
        self._t = None

    def _loop(self):
        try:
            import pynvml as nv

            nv.nvmlInit()
            vis = os.environ.get("CUDA_VISIBLE_DEVICES")
            idx = int(vis.split(",")[self.index]) if vis and vis.split(",")[self.index].isdigit() else self.index
            h = nv.nvmlDeviceGetHandleByIndex(idx)
            self.max_mhz = nv.nvmlDeviceGetMaxClockInfo(h, nv.NVML_CLOCK_SM)
            names = {
                "hw_slowdown": getattr(nv, "nvmlClocksThrottleReasonHwSlowdown", 0x8),
                "hw_thermal_slowdown": getattr(nv, "nvmlClocksThrottleReasonHwThermalSlowdown", 0x40),
                "sw_thermal_slowdown": getattr(nv, "nvmlClocksThrottleReasonSwThermalSlowdown", 0x20),
                "sw_power_cap": getattr(nv, "nvmlClocksThrottleReasonSwPowerCap", 0x4),
                "hw_power_brake": getattr(nv, "nvmlClocksThrottleReasonHwPowerBrakeSlowdown", 0x80),
            }
            while not self._stop.is_set():
                self.samples.append(nv.nvmlDeviceGetClockInfo(h, nv.NVML_CLOCK_SM))
                try:
                    r = nv.nvmlDeviceGetCurrentClocksThrottleReasons(h)
                    for k, bit in names.items():
                        if r & bit:
                            self.reasons.add(k)
                except Exception:
                    pass
                time.sleep(self.period)
        except Exception as e:  # NVML missing: fall back to one nvidia-smi query
            self.reasons.add(f"nvml_unavailable:{type(e).__name__}")

    def __enter__(self):
        self._t = threading.Thread(target=self._loop, daemon=True)
        self._t.start()
        return self

    def __exit__(self, *a):
        self._stop.set()
        self._t.join(timeout=2)

    def summary(self):
        return {"sm_mhz": statistics.median(self.samples) if self.samples else None,
                "sm_max_mhz": self.max_mhz, "reasons": sorted(self.reasons), "samples": len(self.samples)}


def parse_args():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--model", default="meta-llama/Llama-2-7b-hf")
    ap.add_argument("--seq-len", type=int, default=4096)
    ap.add_argument("--batch", type=int, default=1, help="per-GPU micro batch (weak scaling)")
    ap.add_argument("--parallelism", default="ddp", choices=("ddp", "fsdp", "tp", "2d"))
    ap.add_argument("--tensor-parallel", type=int, default=None)
    ap.add_argument("--layers", type=int, default=None,
                    help="DEBUG ONLY: truncate the model; such a number is not a valid benchmark value")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="write the last timed step's loss and a seeded sample of the updated weights as .npy files "
                         "(replicated engines only: one GPU, or --parallelism ddp)")
    return ap.parse_args()


def dump_outputs(out_dir, loss, model, per_param=4096):
    """loss.npy + params_sample.npy (float32, < 64 MB for any model this benchmark runs: 4096 values a parameter)."""
    import numpy as np
    import torch

    os.makedirs(out_dir, exist_ok=True)
    np.save(os.path.join(out_dir, "loss.npy"), np.asarray([float(loss)], dtype=np.float32))
    rng = np.random.default_rng(0)
    parts = []
    for _, p in sorted(model.named_parameters(), key=lambda kv: kv[0]):
        flat = p.detach().reshape(-1)
        n = flat.numel()
        idx = np.sort(rng.integers(0, n, per_param)) if n > per_param else np.arange(n)
        parts.append(flat[torch.from_numpy(idx).to(flat.device)].float().cpu())
    np.save(os.path.join(out_dir, "params_sample.npy"), torch.cat(parts).numpy())


L2_NOTE = "per-step working set (>40 GB of weights/grads/activations) far exceeds the 50 MB L2"


def _config(args, dp, tp, par):
    """The benchmark configuration, IDENTICAL for both arms (the driver compares the dicts): what is computed, not
    how.  Implementation details of an arm go under the top-level "engine" key."""
    strat = {"ddp": "ddp+zero1", "fsdp": "fsdp", "tp": "tp", "2d": "fsdp x tp"}[par]
    mesh = f"dp{dp}" if tp == 1 else f"dp{dp}xtp{tp}"
    return {"model": args.model + (f"[layers={args.layers}]" if args.layers else ""),
            "global_batch": dp * args.batch, "seq_len": args.seq_len, "parallelism": f"{mesh} ({strat})",
            "optimizer": "AdamW, bf16 parameters and states", "l2": L2_NOTE}


def _dist_max(x: float, device) -> float:
    import torch
    import torch.distributed as dist

    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        t = torch.tensor([x], dtype=torch.float64, device=device)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t.item())
    return x


def _barrier_sync(device):
    import torch
    import torch.distributed as dist

    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        dist.barrier()
    torch.cuda.synchronize(device)


_T0 = time.time()
_WATCH = {"deadline": None, "stage": "", "thread": None}
# Stage budgets (seconds).  Their SUM stays below the driver's per-N limit, so a wedged run always leaves a
# diagnosis (stacks + signal-pad state) and exits by itself instead of being killed silently from outside.
BUDGET = {"import": 200, "build": 200, "warmup": 100, "timed": 100, "e2e": 100, "teardown": 60}
for _kv in filter(None, os.environ.get("DTG_BENCH_BUDGET", "").split(",")):  # e.g. "build=90,warmup=40" (debug sessions)
    BUDGET[_kv.split("=")[0]] = int(_kv.split("=")[1])


def _post_mortem(stage):
    """Runs on the watchdog thread when a stage overran: every thread's Python stack, then (best effort, on a side
    stream so it works while a kernel is spinning) the NVLink signal-pad state of every live symmetric group."""
    import faulthandler

    rank = os.environ.get("RANK", "0")
    sys.stderr.write(f"[bench rank {rank}] WATCHDOG: stage '{stage}' exceeded its budget; dumping stacks and exiting\n")
    sys.stderr.flush()
    try:
        faulthandler.dump_traceback(file=sys.__stderr__, all_threads=True)
    except Exception:
        pass
    try:
        symm = sys.modules.get("distributed_training_guide_b200.parallel.symm")  # only if the engine got that far
        for line in (symm.post_mortem(timeout_s=5.0) if symm is not None else []):
            sys.stderr.write(f"[bench rank {rank}] {line}\n")
    except Exception as e:  # pragma: no cover - diagnostics only
        sys.stderr.write(f"[bench rank {rank}] (no signal-pad state: {e!r})\n")
    sys.stderr.flush()
    os._exit(3)


_PROGRESS = {"ticks": 0, "t": None, "engine": None, "reported": False}


def _tick():
    _PROGRESS["ticks"] += 1
    _PROGRESS["t"] = time.time()


def _stall_report(idle_s):
    """A step loop has not moved for a while although its stage budget is not used up yet: say where the host is
    (stacks) and how far the device got (event queries only — nothing here can block behind a wedged kernel)."""
    import faulthandler

    rank = os.environ.get("RANK", "0")
    w = sys.__stderr__
    w.write(f"[bench rank {rank}] STALL: no step completed for {idle_s:.0f} s in stage '{_WATCH['stage']}' "
            f"(after {_PROGRESS['ticks']} steps)\n")
    try:
        import torch

        eng = _PROGRESS["engine"]
        w.write(f"[bench rank {rank}] compute stream idle: {torch.cuda.current_stream(eng.device).query()}\n")
        e = getattr(eng.model, "engine", None)
        if e is not None and hasattr(e, "describe_progress"):
            w.write(f"[bench rank {rank}] {e.describe_progress()}\n")
        symm = sys.modules.get("distributed_training_guide_b200.parallel.symm")
        for line in (symm.post_mortem(timeout_s=3.0) if symm is not None else []):
            w.write(f"[bench rank {rank}] {line}\n")
        ms = torch.cuda.memory_stats(eng.device)
        w.write(f"[bench rank {rank}] allocator: reserved {ms.get('reserved_bytes.all.peak', 0) / 1e9:.1f} GB peak, "
                f"alloc retries {ms.get('num_alloc_retries', 0)} (a retry = cudaFree of cached blocks = device-wide "
                f"synchronisation while peers spin)\n")
    except Exception as e:  # pragma: no cover - diagnostics only
        w.write(f"[bench rank {rank}] (device state unavailable: {e!r})\n")
    w.flush()
    faulthandler.dump_traceback(file=w, all_threads=True)
    w.flush()


def _watch_loop():
    stall_s = float(os.environ.get("DTG_BENCH_STALL_S", "0") or 0)
    while True:
        time.sleep(0.5)
        d = _WATCH["deadline"]
        if d is not None and time.time() > d:
            _post_mortem(_WATCH["stage"])
        t = _PROGRESS["t"]
        if stall_s and t is not None and not _PROGRESS["reported"] and time.time() - t > stall_s:
            _PROGRESS["reported"] = True
            _stall_report(time.time() - t)


def _stage(msg, budget_s=None):
    """Progress line on stderr (rank 0, or every rank with DTG_BENCH_VERBOSE=1) and, with ``budget_s``, a watchdog:
    if the next stage does not report within that many seconds the process dumps a post-mortem and exits."""
    rank = os.environ.get("RANK", "0")
    if rank == "0" or os.environ.get("DTG_BENCH_VERBOSE"):
        print(f"[bench rank {rank} +{time.time() - _T0:6.1f}s] {msg}", file=sys.stderr, flush=True)
    _WATCH["stage"] = msg
    _WATCH["deadline"] = (time.time() + budget_s) if budget_s else None
    if budget_s and _WATCH["thread"] is None and not os.environ.get("DTG_BENCH_NO_WATCHDOG"):
        _WATCH["thread"] = threading.Thread(target=_watch_loop, daemon=True, name="bench-watchdog")
        _WATCH["thread"].start()


def run_b200(args):
    _stage("importing torch", budget_s=BUDGET["import"])
    try:  # a rank killed from outside (torchrun tearing the job down after a peer failed) still says where it was
        import faulthandler
        import signal

        faulthandler.register(signal.SIGTERM, file=sys.__stderr__, all_threads=True, chain=True)
    except Exception:
        pass
    if int(os.environ.get("WORLD_SIZE", "1")) > 1:
        os.environ.setdefault("CUDA_MODULE_LOADING", "EAGER")  # see distributed_training_guide_b200/__init__.py
    os.environ.setdefault("DTG_DIST_TIMEOUT_S", "150")       # a wedged collective aborts with a stack, well inside
    os.environ.setdefault("TORCH_NCCL_DUMP_ON_TIMEOUT", "1")  # the driver's per-N limit
    import torch

    from distributed_training_guide_b200 import _ext
    from distributed_training_guide_b200.engine import TrainEngine

    world = int(os.environ.get("WORLD_SIZE", "1"))
    assert world == args.gpus, f"--gpus {args.gpus} but WORLD_SIZE={world}: launch with torchrun for N>1"
    par = args.parallelism if world > 1 else "single"
    if args.dump_outputs and par not in ("single", "ddp"):
        # fsdp / tp / 2d ranks hold shards or rotating slots, not the parameters a caller of step() would see
        raise SystemExit(f"--dump-outputs needs a replicated engine (one GPU or --parallelism ddp), not {par}")
    _stage(f"building the {par} engine on {world} GPU(s) (process group, NVLink symmetric memory, model)", budget_s=BUDGET["build"])
    eng = TrainEngine.create(args.model, parallelism=par, batch_size=args.batch, seq_length=args.seq_len,
                             tensor_parallel=args.tensor_parallel, num_layers=args.layers)
    dev = eng.device
    rank = eng.env.rank
    # a fresh random batch for every step of the run (nothing is ever seen twice, so the loss stays at the
    # ln(V) of real from-scratch pretraining instead of collapsing by memorisation)
    n_dev = args.warmup + 1 + args.steps
    n_host = 1 + args.steps
    host_batches = [eng.synthetic_batch(seed=n_dev + i) for i in range(n_host)]
    dev_batches = [{k: v.to(dev) for k, v in eng.synthetic_batch(seed=i, pinned=False).items()} for i in range(n_dev)]
    h2d_bytes = sum(v.numel() * v.element_size() for v in host_batches[0].values())

    eng.phase_timing = bool(os.environ.get("DTG_PHASE_TIMING"))
    ddp_engine = getattr(eng.model, "engine", None) or getattr(eng.strategy, "engine", None)
    if world > 1 and hasattr(ddp_engine, "measure_tail"):
        ddp_engine.measure_tail = True   # two CUDA events per step: exposed communication = comm stream past backward
    _stage(f"engine ready; {args.warmup} warm-up steps", budget_s=BUDGET["warmup"] + 2 * args.warmup)
    _PROGRESS["engine"] = eng
    _tick()
    for i in range(args.warmup):
        eng.step(dev_batches[i])
        if os.environ.get("DTG_BENCH_SYNC_WARMUP"):  # debug: one step at a time, so a stall report names the step
            torch.cuda.synchronize(dev)
        _tick()
    torch.cuda.synchronize(dev)
    _PROGRESS["t"] = None
    eng.strategy.check_health()
    if os.environ.get("DTG_CPU_PROFILE") and rank == 0:  # host-side cost of one step (diagnostics)
        import cProfile
        import io
        import pstats

        torch.cuda.synchronize(dev)
        pr = cProfile.Profile()
        t0 = time.perf_counter()
        pr.enable()
        eng.step(dev_batches[args.warmup])
        pr.disable()
        host_ms = 1000 * (time.perf_counter() - t0)
        torch.cuda.synchronize(dev)
        buf = io.StringIO()
        pstats.Stats(pr, stream=buf).sort_stats("cumulative").print_stats(45)
        with open(os.environ["DTG_CPU_PROFILE"], "w") as fp:
            fp.write(f"host time to enqueue one step: {host_ms:.1f} ms\n" + buf.getvalue())
    elif os.environ.get("DTG_CPU_PROFILE"):
        eng.step(dev_batches[args.warmup])
    # ---- region 1: device-timed steps, batch resident on the GPU --------------------------------
    _stage(f"timing {args.steps} steps (device events)", budget_s=BUDGET["timed"] + 2 * args.steps)
    _barrier_sync(dev)
    l0 = _ext.launch_count()
    with ClockSampler(dev.index or 0) as clocks:
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        _tick()
        for i in range(args.steps):
            loss = eng.step(dev_batches[args.warmup + 1 + i])
        e.record()
        _barrier_sync(dev)
    _PROGRESS["t"] = None
    eng.strategy.check_health()   # a device-side barrier that timed out inside the timed region invalidates it: fail loudly
    launches = _ext.launch_count() - l0
    ms_dev = _dist_max(s.elapsed_time(e), dev) / args.steps
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, loss, eng.model)
    _stage(f"device-timed region: {ms_dev:.2f} ms/step = {1000.0 * eng.tokens_per_step / ms_dev:.0f} tokens/s "
           f"(interim; the JSON line follows the end-to-end region); reserved "
           f"{torch.cuda.max_memory_reserved(dev) / 1e9:.1f} GB, alloc retries "
           f"{int(torch.cuda.memory_stats(dev).get('num_alloc_retries', 0))}")
    # ---- region 2: end to end through the public API: pinned H2D every step + loss D2H every step ---
    _stage(f"timing {args.steps} steps end to end (pinned H2D + loss D2H every step)", budget_s=BUDGET["e2e"] + 2 * args.steps)
    eng.step(host_batches[args.steps])
    _barrier_sync(dev)
    _tick()
    s2, e2 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0 = time.perf_counter()
    s2.record()
    last = 0.0
    for i in range(args.steps):
        loss = eng.step(host_batches[i])
        last = loss.item()  # 4-byte device->host read of the step's result
        _tick()             # (stall reporter: this loop synchronises every step, so a missing tick is a real stall)
    e2.record()
    _PROGRESS["t"] = None
    _barrier_sync(dev)
    wall_ms = 1000 * (time.perf_counter() - t0)
    eng.strategy.check_health()
    ms_e2e = _dist_max(max(s2.elapsed_time(e2), wall_ms), dev) / args.steps

    tokens = eng.tokens_per_step
    value = 1000.0 * tokens / ms_dev
    dp = eng.strategy.dp_size
    tp = getattr(eng.strategy, "tp_size", 1)
    pname = PARALLELISM_NAMES[par]
    par_str = "single" if world == 1 else (f"dp{dp}" if par in ("ddp", "fsdp") and tp == 1 else f"dp{dp}xtp{tp}")
    out = {
        "metric": METRIC, "value": value, "unit": "tokens/s", "n_gpus": world, "steps": args.steps,
        "warmup": args.warmup, "ms_per_step": ms_dev, "higher_is_better": True, "scaling": "weak",
        "vs_baseline": None, "dtype": "bf16", "data": "synthetic tokens, random-init weights",
        "impl": "b200",
        "config": _config(args, dp, tp, args.parallelism),
        "engine": f"{par_str} ({pname}): distributed_training_guide_b200 {type(eng.strategy).__name__}",
        "clocks": clocks.summary(),
        "e2e": {"value": 1000.0 * tokens / ms_e2e, "unit": "tokens/s", "ms_per_step": ms_e2e,
                "h2d_bytes_per_step": h2d_bytes, "d2h_bytes_per_step": 4},
        "gpu_launches": int(launches),
        **({"exposed_comm_ms": ddp_engine.exposed_comm_ms(last_steps=2 * args.steps)}
           if world > 1 and hasattr(ddp_engine, "exposed_comm_ms") else {}),
        "final_loss": last,
        **({"phases_ms": eng.phase_times_ms(last_n=args.steps)} if eng.phase_timing else {}),
        **({"comm_trace": eng.model.engine.comm_trace_summary(last_steps=args.steps)}
           if getattr(getattr(eng.model, "engine", None), "trace", None) else {}),
        "peak_alloc_gb": torch.cuda.max_memory_allocated(dev) / 1e9,
        "peak_reserved_gb": torch.cuda.max_memory_reserved(dev) / 1e9,
        "alloc_retries": int(torch.cuda.memory_stats(dev).get("num_alloc_retries", 0)),
    }
    if rank == 0:
        print(json.dumps(out), flush=True)
    _stage("done; tearing down", budget_s=BUDGET["teardown"])
    eng.close()
    from distributed_training_guide_b200.parallel.bootstrap import shutdown

    _barrier_sync(dev)
    shutdown()
    _stage("exit")


def main():
    args = parse_args()
    run_b200(args)


if __name__ == "__main__":
    main()
