"""Phase timers.

``LocalTimer`` keeps the reference's API (``01-single-gpu/train_llm.py:260-286``): a context
manager with ``avg_elapsed_ms()`` / ``reset()``.  On CUDA it records *CUDA events* on the
current stream instead of bracketing each phase with two device synchronisations, so the
host keeps running ahead (the reference pays 8 syncs + one ``.item()`` per step, SURVEY.md
§8 #14) and the numbers are device time, as BASELINE.json requires.  Elapsed times are
resolved lazily when ``avg_elapsed_ms()`` is read (once per ``--log-freq`` steps).
"""
from __future__ import annotations

import os
import time
from contextlib import contextmanager

import torch

NVTX = bool(os.environ.get("DTG_NVTX"))


@contextmanager
def nvtx_range(name: str):
    """``DTG_NVTX=1``: NVTX range around a phase / fused path, so a profiler timeline (nsys, ncu --nvtx) shows
    data / forward / backward / update and every bucket or unshard launch by name.  Free when off."""
    on = NVTX and torch.cuda.is_available()
    if on:
        torch.cuda.nvtx.range_push(name)
    try:
        yield
    finally:
        if on:
            torch.cuda.nvtx.range_pop()


class LocalTimer:
    def __init__(self, device: torch.device, sync: bool = False, name: str = ""):
        self.name = name
        self.device = torch.device(device)
        self.is_cuda = self.device.type == "cuda"
        self.sync = sync  # reference-style host-synchronous timing (used by diagnostics)
        self.measurements = []  # ms floats (cpu) or (start_evt, end_evt) pairs (cuda)
        self._start = None

    def _synchronize(self):
        if self.is_cuda:
            torch.cuda.synchronize(self.device)

    def __enter__(self):
        if NVTX and self.is_cuda and self.name:
            torch.cuda.nvtx.range_push(self.name)
        if self.is_cuda and not self.sync:
            self._start = torch.cuda.Event(enable_timing=True)
            self._start.record()
        else:
            self._synchronize()
            self._start = time.perf_counter()
        return self

    def __exit__(self, exc_type, exc, tb):
        if NVTX and self.is_cuda and self.name:
            torch.cuda.nvtx.range_pop()
        if tb is None:
            if self.is_cuda and not self.sync:
                end = torch.cuda.Event(enable_timing=True)
                end.record()
                self.measurements.append((self._start, end))
            else:
                self._synchronize()
                self.measurements.append(1000.0 * (time.perf_counter() - self._start))
        self._start = None

    def _resolve(self):
        out = []
        for m in self.measurements:
            if isinstance(m, tuple):
                m[1].synchronize()
                out.append(m[0].elapsed_time(m[1]))
            else:
                out.append(m)
        self.measurements = out
        return out

    def avg_elapsed_ms(self) -> float:
        vals = self._resolve()
        return sum(vals) / max(len(vals), 1)

    def total_elapsed_ms(self) -> float:
        return sum(self._resolve())

    def reset(self):
        self.measurements = []
        self._start = None


def device_time_ms(fn, warmup=3, iters=10, flush_l2=True):
    """CUDA-event timing of ``fn`` per the profiling recipe: warm-up, L2 flush between
    iterations (a 256 MiB write > the 50 MB L2), synchronise on both sides."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    scratch = torch.empty(256 << 20, dtype=torch.uint8, device="cuda") if flush_l2 else None
    times = []
    for _ in range(iters):
        if scratch is not None:
            scratch.zero_()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        e.synchronize()
        times.append(s.elapsed_time(e))
    times.sort()
    return times[len(times) // 2], times
